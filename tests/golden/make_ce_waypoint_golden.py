"""Generates tests/golden/small_ce_waypoint.pt by running the UNMODIFIED waypoint predictor of the VLN-CE policy
(bevbert_ce/vlnce_baselines/waypoint_pred/TRM_net.py::BinaryDistPredictor_TRM over transformer/waypoint_bert.py and the
reference's own copy of pytorch_transformer/modeling_bert.py) and its heatmap NMS (waypoint_pred/utils.py::nms), from
the reference checkout located by oracle/ref_shim.py (env BEVBERT_REFERENCE):

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_ce_waypoint_golden.py

TRM_net.py imports `vlnce_baselines.waypoint_pred.utils` and `pytorch_transformers.BertConfig`, so the modules are
imported through stub parent packages whose `__path__` points at the reference directories (their `__init__` never
runs), a `pytorch_transformers` stub that exposes the reference copy's BertConfig, and stubs for boto3, requests,
botocore and tqdm, which the copy's file_utils.py imports for its model downloader (never called here).  Weights are
bevbert_b200.synth.waypoint_state(SEED); inputs are seeded depth features at B = 1 and 3, run in fp32 on the CPU in eval
mode.

Stored (data only): the state_dict key -> shape map in order; of the logits (B, 120, 12) the first 12 values of rows 0,
5 and 119, every row's norm and the projection on PROBES seeded directions; the reference `nms` output on the policy's
wrapped, softmaxed heatmaps of those logits and on constructed cases (ties, negatives, NaN, +-0, other H, W, sigma and
k); and the suppression footprint of every centre of the policy's 122 x 12 map with sigma = (7, 5)."""
import importlib
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT]

from bevbert_b200 import synth  # noqa: E402
from oracle import ref_shim  # noqa: E402

SEED, FEAT_SEED, PROBES = 21, 22, 4
BATCHES = (1, 3)
POLICY = dict(max_predictions=5, sigma=(7.0, 5.0))
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "small_ce_waypoint.pt")


def depth_feats(B, seed=FEAT_SEED):
    """seeded depth-encoder outputs of 12 B views, (12 B, 128, 4, 4), ReLU-like (non-negative)"""
    return synth.det_uniform((12 * B, 128, 4, 4), seed, 100 + B, 0.0, 1.0)


def probes(shape):
    return synth.det_uniform((PROBES,) + tuple(shape), 78, 1, -1.0, 1.0).double()


def summarize(logits):
    x = logits.double()
    return {"first": x[:, [0, 5, 119], :12], "row_norm": x.norm(dim=-1),
            "proj": torch.einsum("bac,pac->bp", x, probes(x.shape[1:]))}


def policy_heatmap(logits):
    """Policy_ViewSelection_BEV.py:212-220: softmax over all 1440 cells, then one wrapped row at each end ->
    (B, 1, 122, 12)"""
    B = logits.shape[0]
    x = torch.softmax(logits.reshape(B, -1), dim=1).reshape(B, 120, 12)
    return torch.cat((x[:, -1:], x, x[:, :1]), dim=1).unsqueeze(1)


def nms_cases():
    """constructed NMS inputs: name -> (pred (B, 1, H, W) fp32, max_predictions, sigma)"""
    g = torch.Generator().manual_seed(5)
    cases = {}
    r = torch.rand(2, 1, 122, 12, generator=g)
    cases["policy_random"] = (r, 5, (7.0, 5.0))
    t = torch.zeros(2, 1, 122, 12)
    t[0, 0, 30, [2, 9]] = 0.5                           # ties: the lower flat index wins
    t[0, 0, 90, 4] = 0.5
    t[1, 0, [3, 60, 118], 0] = 0.25
    cases["ties"] = (t, 5, (7.0, 5.0))
    cases["all_equal"] = (torch.full((1, 1, 122, 12), 0.125), 5, (7.0, 5.0))
    cases["negatives"] = (-torch.rand(2, 1, 122, 12, generator=g) - 0.1, 5, (7.0, 5.0))
    m = torch.rand(2, 1, 122, 12, generator=g) - 0.5   # mixed signs: suppressed negatives become -0.0
    cases["mixed_signs"] = (m, 8, (2.0, 3.0))
    n = torch.rand(2, 1, 122, 12, generator=g)
    n[0, 0, 40, 7] = float("nan")
    n[0, 0, 100, 1] = float("nan")
    n[1, 0, 5, 5] = float("inf")                        # inf * 0 = NaN once suppressed
    cases["nan_inf"] = (n, 5, (7.0, 5.0))
    z = torch.zeros(1, 1, 122, 12)
    z[0, 0, ::3] = -0.0                                 # -0.0 and +0.0 compare equal
    z[0, 0, 50, 6] = -0.0
    cases["signed_zeros"] = (z, 5, (7.0, 5.0))
    cases["all_negative_zero"] = (torch.full((1, 1, 16, 8), -0.0), 3, (1.0, 1.0))
    q = -torch.rand(2, 1, 122, 12, generator=g) - 0.5  # one positive patch in a negative map: once the patch is
    q[:, 0, 20:31] = torch.rand(2, 11, 12, generator=g) * 0.5 + 0.1   # suppressed to +0, later rounds pick
    q[0, 0, 25, 6] = 1.0                                               # suppressed cells (the first of them is
    q[1, 0, 20, 0] = 1.0                                               # the peak itself in row 1)
    cases["repick_suppressed"] = (q, 5, (7.0, 5.0))
    for i, (B, H, W, k, sig) in enumerate([(3, 24, 48, 10, (1.0, 1.0)), (2, 7, 5, 4, (1.5, 0.5)),
                                           (2, 122, 12, 12, (3.0, 2.0)), (1, 1, 1, 3, (0.0, 0.0)),
                                           (2, 32, 64, 6, (10.0, 4.0)), (3, 122, 12, 0, (7.0, 5.0)),
                                           (2, 13, 7, 9, (0.3, 2.7)), (1, 60, 60, 20, (5.0, 7.0))]):
        cases["shape_%d" % i] = (torch.rand(B, 1, H, W, generator=g) * 2 - 0.25, k, sig)
    return cases


def footprint_table(utils):
    """the cells one nms round suppresses around every centre ix of the policy's 122 x 12 map, sigma = (7, 5), from
    the reference's `neighborhoods` on the centre nms builds (x = ix % W, y = ix / W) -> (1464, 122 * 12) bool, True =
    suppressed, packed 8 cells to a byte (numpy.packbits along the last axis)."""
    import numpy as np
    H, W = 122, 12
    ix = torch.arange(H * W)
    mu = torch.stack([ix % W, ix / W], dim=1).float()
    g = utils.neighborhoods(mu, W, H, POLICY["sigma"]).bool().reshape(H * W, H * W)
    return torch.from_numpy(np.packbits(g.numpy(), axis=-1))


def _pkg(name, path=None):
    m = types.ModuleType(name)
    if path is not None:
        m.__path__ = [path]
    sys.modules[name] = m
    return m


def load_reference():
    """-> (TRM_net module, utils module) of the unmodified reference"""
    base = os.path.join(ref_shim.REF_ROOT, "bevbert_ce", "vlnce_baselines")
    if not os.path.isdir(base):
        raise RuntimeError("CE reference tree not found under %s" % ref_shim.REF_ROOT)
    sys.dont_write_bytecode = True
    wp = os.path.join(base, "waypoint_pred")
    for name in ("boto3", "requests", "tqdm"):
        _pkg(name)
    sys.modules["tqdm"].tqdm = None
    _pkg("botocore")
    _pkg("botocore.exceptions").ClientError = type("ClientError", (Exception,), {})
    _pkg("vlnce_baselines", base)
    _pkg("vlnce_baselines.waypoint_pred", wp)
    _pkg("vlnce_baselines.waypoint_pred.transformer", os.path.join(wp, "transformer"))
    _pkg("vlnce_baselines.waypoint_pred.transformer.pytorch_transformer",
         os.path.join(wp, "transformer", "pytorch_transformer"))
    mb = importlib.import_module("vlnce_baselines.waypoint_pred.transformer.pytorch_transformer.modeling_bert")
    _pkg("pytorch_transformers").BertConfig = mb.BertConfig
    trm = importlib.import_module("vlnce_baselines.waypoint_pred.TRM_net")
    utils = importlib.import_module("vlnce_baselines.waypoint_pred.utils")
    for m in (mb, trm, utils):
        assert m.__file__.startswith(base), m.__file__
    return trm, utils


def main():
    trm, utils = load_reference()
    torch.manual_seed(0)
    net = trm.BinaryDistPredictor_TRM(device="cpu")
    net.load_state_dict(synth.waypoint_state(SEED))
    net.requires_grad_(False).eval()
    out = {"keys": [(k, tuple(v.shape)) for k, v in net.state_dict().items()], "seed": SEED, "feat_seed": FEAT_SEED,
           "attention_mask": utils.get_attention_mask(num_imgs=12, neighbor=1).clone()}
    cases = {}
    for B in BATCHES:
        dep = depth_feats(B)
        rgb = torch.zeros(12 * B, 512)                  # only its size(0) is read
        with torch.no_grad():
            logits = net(rgb, dep)
        out["logits_B%d" % B] = summarize(logits)
        cases["policy_B%d" % B] = (policy_heatmap(logits), POLICY["max_predictions"], POLICY["sigma"])
    cases.update(nms_cases())
    out["nms"] = {name: {"pred": p.clone(), "k": k, "sigma": s,
                         "out": utils.nms(p.clone(), max_predictions=k, sigma=s, gaussian=False)}
                  for name, (p, k, s) in cases.items()}
    out["footprint"] = footprint_table(utils)
    torch.save(out, OUT)
    print("wrote %s" % OUT)


if __name__ == "__main__":
    main()
