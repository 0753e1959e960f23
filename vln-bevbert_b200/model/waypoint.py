"""The VLN-CE waypoint predictor and its heatmap NMS on the H100 kernels, forward only: the policy's `waypoint` mode
(bevbert_ce/vlnce_baselines/models/Policy_ViewSelection_BEV.py:194-224) over waypoint_pred/TRM_net.py
BinaryDistPredictor_TRM and waypoint_pred/utils.py nms.

`BinaryDistPredictor_TRM` has the reference class's constructor, parameter names, shapes and order (the unused
`visual_merge` and `mergefeats_LayerNorm` included, so a reference checkpoint loads strictly); `WaypointRunner` runs the
same forward over the parameters of any module with that layout, such as the reference's own instance
(graphs.install_ce_waypoint_predictor).  Per call, on N = 12 B views:
    depth features (N, 128, 4, 4) flattened -> GEMM 2048 -> 768 with the ReLU epilogue -> 2 post-LN BERT layers
    (blocks.BertLayerImpl: erf-GELU, eps 1e-12) with the (B, 12, 12) neighbour bias, 0 between views at most one
    apart around the panorama and -10000 otherwise -> GEMM 768 -> 768 with ReLU -> GEMM 768 -> 120 in fp32 ->
    (B, 120, 12), rolled up by HEATMAP_OFFSET rows.
Weights are read through WeightCache shadows, re-made when a parameter's version or storage changes.  The trainer keeps
the predictor frozen and in eval mode; a call in training mode raises (the reference applies dropout there), and so
does a call with grad enabled while a parameter requires grad, because nothing here runs backward.  Autocast is
disabled inside the call, so the trainer's autocast() changes no bit of the outputs.

`nms` is the reference's nms(pred, max_predictions, sigma, gaussian=False) in one launch (bb_waypoint_nms).
"""
import numpy as np
import torch
from torch import nn

from .. import _lib
from .. import blocks
from .. import kernels as K

NUM_IMGS, NUM_ANGLES, NUM_CLASSES, HEATMAP_OFFSET = 12, 120, 12, 5
HIDDEN, HEADS, FFN, LN_EPS = 768, 12, 3072, 1e-12
NMS_MAX_CELLS = 8192        # H * W of one map in bb_waypoint_nms; the policy's is 122 x 12


def nms(pred, max_predictions=10, sigma=(1.0, 1.0), gaussian=False):
    """waypoint_pred/utils.py nms on the GPU: pred (B, 1, H, W) fp32 CUDA -> a fresh (B, 1, H, W) fp32 map holding
    pred at the cells picked by `max_predictions` rounds of argmax and box suppression, negatives clamped to 0, and 0
    elsewhere.  Bit-identical to the reference on the CPU.  gaussian=True (which the policy never passes) raises."""
    if gaussian:
        raise NotImplementedError("bb_waypoint_nms implements gaussian=False, the policy's call")
    if pred.dtype != torch.float32:
        raise TypeError("pred must be float32, got %s" % pred.dtype)
    if not pred.is_cuda:
        raise RuntimeError("pred must be a CUDA tensor (the hot path has no CPU implementation)")
    if pred.dim() != 4 or pred.shape[1] != 1:
        raise ValueError("pred must be (B, 1, H, W), got %s" % (tuple(pred.shape),))
    B, _, H, W = pred.shape
    if H * W > NMS_MAX_CELLS:
        raise ValueError("H * W = %d exceeds the %d cells bb_waypoint_nms holds in shared memory" % (H * W, NMS_MAX_CELLS))
    x = pred.contiguous()
    out = torch.empty_like(x)
    if B == 0:
        return out
    _lib.check(_lib.load().bb_waypoint_nms(x.data_ptr(), B, H, W, float(sigma[0]), float(sigma[1]),
                                           max(0, int(max_predictions)), out.data_ptr(), K._stream()),
               "bb_waypoint_nms")
    return out


def neighbour_mask():
    """(12, 12) 0/1, utils.get_attention_mask(12, neighbor=1): row i is 1 at views i - 1, i and i + 1 (mod 12)"""
    i = np.arange(NUM_IMGS)
    d = (i[:, None] - i[None, :]) % NUM_IMGS
    return torch.from_numpy(((d <= 1) | (d == NUM_IMGS - 1)).astype(np.int64))


class WaypointRunner:
    """The kernels' forward over `module`, laid out as TRM_net.py's BinaryDistPredictor_TRM (visual_fc_depth.1,
    waypoint_TRM.bert.encoder.layer[i].{attention.self.{query,key,value}, attention.output.{dense,LayerNorm},
    intermediate.dense, output.{dense,LayerNorm}}, vis_classifier.{0,2}).  `owner` (default `module`) is the module
    whose train / eval mode the caller goes by."""

    def __init__(self, module, owner=None):
        self.m, self.owner = module, owner if owner is not None else module
        fc, cls = module.visual_fc_depth[1], module.vis_classifier
        got = (tuple(fc.weight.shape), tuple(cls[0].weight.shape), tuple(cls[2].weight.shape))
        if got != ((HIDDEN, 2048), (HIDDEN, HIDDEN), (NUM_ANGLES, HIDDEN)):
            raise ValueError("expected the predictor's 768-wide layout (hidden_dim=768, n_classes=12), got %s" % (got,))
        self.layers = list(module.waypoint_TRM.bert.encoder.layer)
        self.rt = blocks.Runtime()
        self.layer = blocks.BertLayerImpl(self.rt, HEADS, LN_EPS)      # eval mode: no dropout
        self._bias = {}
        self._sig = None

    @property
    def training(self):
        return self.owner.training

    def parameters(self):
        return self.m.parameters()

    def changed(self):
        """True when a parameter's storage or version moved since the previous call of this method."""
        sig = tuple((p.data_ptr(), p._version) for p in self.m.parameters())
        moved, self._sig = sig != self._sig, sig
        return moved

    def check_call(self):
        if self.training:
            raise RuntimeError("the waypoint predictor runs in eval mode only (the reference applies dropout 0.3 / 0.1 "
                               "in training mode): call .eval() on it, as the trainer does")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.m.parameters()):
            raise RuntimeError("the waypoint predictor runs forward only: call it under torch.no_grad() or freeze its "
                               "parameters (requires_grad_(False)), as the trainer does")

    def bias(self, B, device):
        """the (B, 12, 12) fp32 additive attention mask, (1 - neighbour_mask) * -10000, built once per (B, device)"""
        key = (B, device)
        if key not in self._bias:
            m = neighbour_mask().to(device=device, dtype=torch.float32)
            self._bias[key] = ((1.0 - m) * -10000.0).expand(B, NUM_IMGS, NUM_IMGS).contiguous()
        return self._bias[key]

    @staticmethod
    def check_inputs(rgb_feats, depth_feats):
        """B = rgb_feats.size(0) // 12, as the reference takes it (rgb_feats is otherwise unused); depth_feats must
        hold the 12 B views, (12 B, 128, 4, 4) fp32 or fp16 (the depth encoder under autocast) -> depth_feats"""
        B = rgb_feats.size(0) // NUM_IMGS
        if B == 0 or depth_feats.dim() == 0 or depth_feats.shape[0] != B * NUM_IMGS or depth_feats[0].numel() != 2048:
            raise ValueError("expected depth features (12 B, 128, 4, 4) with B = rgb_feats.size(0) // 12 = %d, got %s"
                             % (B, tuple(depth_feats.shape)))
        if depth_feats.dtype not in (torch.float32, torch.float16):
            raise TypeError("depth_feats must be float32 or float16, got %s" % depth_feats.dtype)
        return depth_feats

    def __call__(self, rgb_feats, depth_feats):
        """BinaryDistPredictor_TRM.forward -> logits (B, 120, 12), a fresh fp32 tensor"""
        self.check_call()
        return self.logits(self.check_inputs(rgb_feats, depth_feats))

    def logits(self, depth_feats):
        """the forward on checked depth features (12 B, 128, 4, 4)"""
        self.check_call()
        with torch.autocast("cuda", enabled=False), torch.no_grad():
            return self._forward(depth_feats, depth_feats.shape[0] // NUM_IMGS)

    def _forward(self, dep, B):
        wc, N = self.rt.wc, B * NUM_IMGS
        x = dep.reshape(N, 2048)
        if x.dtype != torch.float32:
            x = x.float()                       # fp16 depth features under the trainer's autocast
        fc, cls = self.m.visual_fc_depth[1], self.m.vis_classifier
        h, _ = blocks.lin_fwd(K.cast_to_act(x), wc.get(fc.weight), fc.bias.detach(), act=K.ACT_RELU)
        bias = self.bias(B, dep.device)
        h = h.view(B, NUM_IMGS, HIDDEN)
        for L in self.layers:
            a, o = L.attention, L.output
            p = [a.self.query.weight, a.self.query.bias, a.self.key.weight, a.self.key.bias, a.self.value.weight,
                 a.self.value.bias, a.output.dense.weight, a.output.dense.bias, a.output.LayerNorm.weight,
                 a.output.LayerNorm.bias, L.intermediate.dense.weight, L.intermediate.dense.bias, o.dense.weight,
                 o.dense.bias, o.LayerNorm.weight, o.LayerNorm.bias]
            h = self.layer.fwd({}, (h, None, bias), p)
        h, _ = blocks.lin_fwd(h.reshape(N, HIDDEN), wc.get(cls[0].weight), cls[0].bias.detach(), act=K.ACT_RELU)
        logits, _ = blocks.lin_fwd(h, wc.get(cls[2].weight), cls[2].bias.detach(), out_f32=True)
        # (B, 120, 12) rows r -> r - HEATMAP_OFFSET (mod 120): TRM_net.py's cat((v[:, 5:], v[:, :5]), 1)
        return torch.roll(logits.view(B, NUM_ANGLES, NUM_CLASSES), -HEATMAP_OFFSET, dims=1)


# ------------------------------------------------------------------------------------------------ containers
class _LayerNorm(nn.Module):
    """modeling_bert.py's BertLayerNorm parameters (weight, bias)"""

    def __init__(self, hidden):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden))
        self.bias = nn.Parameter(torch.zeros(hidden))


def _container(**children):
    m = nn.Module()
    for k, v in children.items():
        setattr(m, k, v)
    return m


def _bert_layer():
    """CaptionBertLayer's parameters under its names and in its registration order"""
    D = HIDDEN
    attention = _container(self=_container(query=nn.Linear(D, D), key=nn.Linear(D, D), value=nn.Linear(D, D),
                                           dropout=nn.Dropout(0.1)),
                           output=_container(dense=nn.Linear(D, D), LayerNorm=_LayerNorm(D), dropout=nn.Dropout(0.3)))
    return _container(attention=attention, intermediate=_container(dense=nn.Linear(D, FFN)),
                      output=_container(dense=nn.Linear(FFN, D), LayerNorm=_LayerNorm(D), dropout=nn.Dropout(0.3)))


class BinaryDistPredictor_TRM(nn.Module):
    """TRM_net.py's BinaryDistPredictor_TRM on the kernels: same constructor, state_dict keys, shapes and order.
    forward(rgb_feats, depth_feats) -> heatmap logits (B, 120, 12) in fp32, B = rgb_feats.size(0) // 12."""

    def __init__(self, hidden_dim=768, n_classes=12, device=None):
        super().__init__()
        self.device = device
        self.num_angles, self.num_imgs, self.n_classes = NUM_ANGLES, NUM_IMGS, NUM_CLASSES
        self.TRM_LAYER, self.TRM_NEIGHBOR, self.HEATMAP_OFFSET = 2, 1, HEATMAP_OFFSET
        self.visual_fc_depth = nn.Sequential(nn.Flatten(), nn.Linear(128 * 4 * 4, hidden_dim), nn.ReLU(True))
        self.visual_merge = nn.Sequential(nn.Linear(hidden_dim * 2, hidden_dim), nn.ReLU(True))
        self.waypoint_TRM = _container(bert=_container(encoder=_container(
            layer=nn.ModuleList([_bert_layer() for _ in range(self.TRM_LAYER)]))), dropout=nn.Dropout(0.3))
        self.mergefeats_LayerNorm = _LayerNorm(hidden_dim)
        self.vis_classifier = nn.Sequential(nn.Linear(hidden_dim, hidden_dim), nn.ReLU(),
                                            nn.Linear(hidden_dim, int(n_classes * (NUM_ANGLES / NUM_IMGS))))
        object.__setattr__(self, "_runner", None)

    @property
    def runner(self):
        if self._runner is None:
            object.__setattr__(self, "_runner", WaypointRunner(self))
        return self._runner

    def forward(self, rgb_feats, depth_feats):
        return self.runner(rgb_feats, depth_feats)
