"""TEST INFRASTRUCTURE ONLY -- oracle for the VLN-CE waypoint predictor and its heatmap NMS (model/waypoint.py).

A functional restatement of BinaryDistPredictor_TRM.forward (bevbert_ce/vlnce_baselines/waypoint_pred/TRM_net.py:62-88,
over transformer/waypoint_bert.py and pytorch_transformer/modeling_bert.py) on a flat state_dict with the predictor's
keys, and of utils.py's `nms` with gaussian=False:

  * `forward(sd, depth_feats, dtype)`: every operation in `dtype` (fp32 or fp64) on the device of the tensors;
  * `forward_fp16(sd, depth_feats)`: the same operations under torch.autocast("cuda", float16) with fp32 weights, the
    reference's dtype flow inside the trainer's `autocast()` (_train_interval): Linear / matmul in fp16, softmax in
    fp32, the additive mask in the parameters' dtype.  scripts/bench_ce_waypoint.py times it as a reference path;
  * `nms(pred, max_predictions, sigma)`: the NMS rounds on the CPU, every value the reference rounds to fp32 rounded
    to fp32 (computed in fp64 first; a single division, subtraction or addition of fp32 values rounded once from fp64
    is the correctly rounded fp32 result), torch.max's tie and NaN rules restated with comparisons.

Pinned against the unmodified reference by tests/golden/small_ce_waypoint.pt (tests/golden/make_ce_waypoint_golden.py).
The product never imports it.
"""
import math

import torch
import torch.nn.functional as F

NUM_IMGS, NUM_ANGLES, NUM_CLASSES, HEATMAP_OFFSET = 12, 120, 12, 5
EPS = 1e-12


def neighbour_mask(n=NUM_IMGS):
    """(n, n) 0/1: key j is a neighbour of query i when they are at most one view apart around the panorama"""
    i = torch.arange(n)
    d = (i[:, None] - i[None, :]) % n
    return ((d <= 1) | (d >= n - 1)).long()


def neighbour_bias(B, dtype=torch.float32, device=None):
    """the additive attention mask WaypointBert builds from it, (B, 1, n, n): 0 for a neighbour, -10000 otherwise"""
    m = neighbour_mask().to(device=device, dtype=dtype)
    return ((1.0 - m) * -10000.0).expand(B, 1, NUM_IMGS, NUM_IMGS)


def _ln(x, sd, k):
    """the TF-style BertLayerNorm of modeling_bert.py (apex absent), operation by operation"""
    u = x.mean(-1, keepdim=True)
    s = (x - u).pow(2).mean(-1, keepdim=True)
    return sd[k + ".weight"] * ((x - u) / torch.sqrt(s + EPS)) + sd[k + ".bias"]


def _lin(x, sd, k):
    return F.linear(x, sd[k + ".weight"], sd[k + ".bias"])


def _forward(sd, x, mask_dtype):
    N = x.shape[0]
    B = N // NUM_IMGS
    h = F.relu(_lin(x.flatten(1), sd, "visual_fc_depth.1")).reshape(B, NUM_IMGS, -1)
    mask = neighbour_bias(B, mask_dtype, x.device)
    D = h.shape[-1]
    nh = D // 64
    for i in range(len([k for k in sd if k.endswith("attention.self.query.weight")])):
        p = "waypoint_TRM.bert.encoder.layer.%d." % i
        q, k, v = (_lin(h, sd, p + "attention.self." + n).view(B, NUM_IMGS, nh, 64).transpose(1, 2)
                   for n in ("query", "key", "value"))
        s = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(64) + mask
        ctx = torch.matmul(torch.softmax(s, dim=-1), v).transpose(1, 2).reshape(B, NUM_IMGS, D)
        a = _ln(_lin(ctx, sd, p + "attention.output.dense") + h, sd, p + "attention.output.LayerNorm")
        f = _lin(a, sd, p + "intermediate.dense")
        f = f * 0.5 * (1.0 + torch.erf(f / math.sqrt(2.0)))
        h = _ln(_lin(f, sd, p + "output.dense") + a, sd, p + "output.LayerNorm")
    y = _lin(F.relu(_lin(h, sd, "vis_classifier.0")), sd, "vis_classifier.2").reshape(B, NUM_ANGLES, NUM_CLASSES)
    return torch.cat((y[:, HEATMAP_OFFSET:], y[:, :HEATMAP_OFFSET]), dim=1)


def forward(sd, depth_feats, dtype=torch.float32):
    """BinaryDistPredictor_TRM.forward in eval mode: depth_feats (12 B, 128, 4, 4) -> logits (B, 120, 12) in dtype"""
    sd = {k: v.to(dtype) for k, v in sd.items()}
    return _forward(sd, depth_feats.to(dtype), dtype)


def forward_fp16(sd, depth_feats):
    """the reference's forward under the trainer's autocast() (fp16) on the GPU, fp32 weights -> fp32 logits"""
    sd = {k: v.float() for k, v in sd.items()}
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        return _forward(sd, depth_feats, torch.float32).float()


# ------------------------------------------------------------------------------------------------ NMS
def _f32(x):
    return x.to(torch.float32).to(torch.float64)


def argmax_rows(v):
    """torch.max(v, dim=1)'s index on (B, n): the first NaN if a row has one, else the first of the largest values
    (-0.0 == +0.0)"""
    nan = torch.isnan(v)
    finite_best = torch.where(nan, torch.full_like(v, -math.inf), v).max(dim=1, keepdim=True).values
    first = lambda m: m.to(torch.int64).argmax(dim=1)     # argmax of 0 / 1 returns the first 1
    return torch.where(nan.any(dim=1), first(nan), first(v == finite_best))


def neighbourhood(ix, H, W, sigma):
    """utils.py `neighborhoods` with gaussian=False at the centres nms builds from flat indices ix (B,):
    x_mu = ix % W, y_mu = fp32(ix / W) -> (B, H, W) bool, True = suppressed"""
    sx, sy = (float(torch.tensor(s, dtype=torch.float32)) for s in sigma)
    ix = ix.to(torch.float64)
    x_mu = torch.remainder(ix, W).view(-1, 1, 1)
    y_mu = _f32(ix / W).view(-1, 1, 1)
    x = torch.arange(W, dtype=torch.float64).view(1, 1, W)
    y = torch.arange(H, dtype=torch.float64).view(1, H, 1)
    xd = _f32(x - x_mu)
    xc = torch.minimum(xd.abs(), _f32(xd + W).abs())
    yd = _f32(y - y_mu)
    return (xc <= sx) & (yd.abs() <= sy)


def nms(pred, max_predictions=10, sigma=(1.0, 1.0)):
    """utils.py nms(pred, max_predictions, sigma, gaussian=False) on pred (B, 1, H, W) fp32 -> (B, 1, H, W) fp32 on the
    CPU"""
    pred = pred.detach().cpu()
    B, _, H, W = pred.shape
    flat = pred.reshape(B, H * W)
    supp = flat.clone()
    out = torch.zeros_like(flat)
    rows = torch.arange(B)
    for _ in range(max_predictions):
        ix = argmax_rows(supp)
        out[rows, ix] = flat[rows, ix]
        keep = (~neighbourhood(ix, H, W, sigma)).to(torch.float32).reshape(B, H * W)
        supp = supp * keep                              # literal multiply: -x * 0 = -0.0, NaN * 0 = inf * 0 = NaN
    out[out < 0] = 0
    return out.view(B, 1, H, W)


def nms_device(pred, max_predictions=10, sigma=(1.0, 1.0)):
    """the reference nms's sequence of torch operations on pred's own device (a max, an index_put with a host-built
    row index, the centre's division, remainder and stack, the box mask, a multiply per round), which
    scripts/bench_ce_waypoint.py times as the reference path.  On a CUDA tensor torch divides by the scalar W as a
    multiply by its fp32 reciprocal, which keeps the policy's rows (W = 12) but is not `nms` above in general."""
    B, _, H, W = pred.shape
    out = torch.zeros_like(pred)
    supp = pred.clone()
    src, dst = pred.reshape(B, -1), out.reshape(B, -1)
    for _ in range(max_predictions):
        ix = supp.reshape(B, -1).max(dim=1)[1]
        rows = torch.arange(B)
        dst[rows, ix] = src[rows, ix]
        mu = torch.stack([ix % W, ix / W], dim=1).float()
        x = torch.arange(W, device=pred.device, dtype=torch.float32).view(1, 1, W)
        y = torch.arange(H, device=pred.device, dtype=torch.float32).view(1, H, 1)
        dx = x - mu[:, 0].view(-1, 1, 1)
        dx = torch.min(dx.abs(), (dx + W).abs())
        dy = y - mu[:, 1].view(-1, 1, 1)
        g = torch.logical_and(dx.abs() <= sigma[0], dy.abs() <= sigma[1]).float()
        supp *= 1 - g.unsqueeze(1)
    out[out < 0] = 0
    return out


def footprint(H=122, W=12, sigma=(7.0, 5.0)):
    """the cells one round suppresses around every centre of an H x W map -> (H W, H W) bool"""
    return neighbourhood(torch.arange(H * W), H, W, sigma).reshape(H * W, H * W)
