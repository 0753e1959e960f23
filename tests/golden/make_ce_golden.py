"""Generates tests/golden/small_ce.pt by running the UNMODIFIED VLN-CE pre-training model
(bevbert_ce/pretrain/pretrain_src/model of the reference checkout located by oracle/ref_shim.py, env BEVBERT_REFERENCE)
on seeded weights and synthetic CE batches:

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_ce_golden.py

The same library-drift shims as oracle/ref_shim.py (torch_scatter stub, transformers init / tying hooks, CPU-only
`.cuda()`, the projector built on the host); none touches the reference's arithmetic.  Both reference trees name their
package `model`, so any `model*` module already imported is dropped before the CE tree is put first on sys.path.

Stored (data only): the reference's state_dict key -> shape map and its named_parameters() order (both in the
reference's order, which its optimizer relies on), and, per task, the per-item losses, the logits, the norm of every
parameter gradient, its projections on PROBES seeded directions (grad_probes: they pin each gradient's direction, not
only its norm) and the full gradients of the CE-specific and a few shared parameters (FULL_GRADS).
The weights (synth.det_init_, seed WEIGHT_SEED) and the batches (synth.make_batch, seed BATCH_SEED) are regenerated bit
for bit from their seeds on any machine, so the file stores the seeds instead of 94 M parameters."""
import importlib
import math
import os
import sys
import types
import zlib

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from bevbert_b200 import synth  # noqa: E402
from bevbert_b200.config import make_ce_config  # noqa: E402
from oracle import ref_shim  # noqa: E402

TASKS = ("mlm", "sap")
WEIGHT_SEED, BATCH_SEED = 3, 7
FULL_GRADS = ["bert.img_embeddings.dep_linear.bias", "bert.img_embeddings.dep_layer_norm.weight",
              "bert.img_embeddings.dep_layer_norm.bias", "bert.img_embeddings.loc_linear.weight",
              "bert.img_embeddings.loc_linear.bias", "bert.img_embeddings.nav_type_embedding.weight",
              "bert.img_embeddings.img_linear.bias", "bert.img_embeddings.layer_norm.weight",
              "bert.embeddings.token_type_embeddings.weight", "bert.local_encoder.bev_pos_embeddings.0.weight",
              "bert.global_encoder.sprel_linear.weight", "sap_fuse_linear.net.3.weight"]


PROBES, PROBE_SEED = 2, 11


def grad_probes(name, shape):
    """(PROBES, *shape) fp64 directions, uniform in [-1, 1), regenerated bit for bit from (PROBE_SEED, name)"""
    stream = zlib.crc32(name.encode())
    return torch.stack([synth.det_uniform(shape, PROBE_SEED, stream * PROBES + k, -1.0, 1.0) for k in range(PROBES)]
                       ).to(torch.float64)


def grad_projections(name, g):
    """[<g, r_k>] over the directions of grad_probes, summed in fp64"""
    r = grad_probes(name, tuple(g.shape))
    return (r * g.detach().to(torch.float64)[None]).reshape(PROBES, -1).sum(1)


def case():
    """(config, synthetic-batch config) of the stored case; the tests rebuild both from here."""
    return make_ce_config(small=True), synth.ce_synth_config(batch_size=2, pano_min=4, pano_max=6, gmap_min=8, gmap_max=8)


def load_ce_modules():
    src = os.path.join(ref_shim.REF_ROOT, "bevbert_ce", "pretrain", "pretrain_src")
    if not os.path.isdir(os.path.join(src, "model")):
        raise RuntimeError("CE reference tree not found under %s" % ref_shim.REF_ROOT)
    sys.dont_write_bytecode = True
    for name in [m for m in sys.modules if m == "model" or m.startswith("model.")]:
        del sys.modules[name]
    sys.path.insert(0, src)
    if "torch_scatter" not in sys.modules:
        stub = types.ModuleType("torch_scatter")
        stub.scatter_mean = ref_shim._scatter_mean
        stub.scatter_max = lambda *a, **k: (_ for _ in ()).throw(NotImplementedError("scatter_max stub"))
        sys.modules["torch_scatter"] = stub
    vilmodel = importlib.import_module("model.vilmodel")
    vilmodel.BertPreTrainedModel.init_weights = lambda self: None
    vilmodel.BertPreTrainedModel._tie_or_clone_weights = lambda self, out, inp: setattr(out, "weight", inp.weight)
    torch.Tensor.cuda = lambda self, *a, **k: self
    pretrain_cmt = importlib.import_module("model.pretrain_cmt")
    bev_utils = importlib.import_module("model.bev_utils")
    assert os.path.dirname(pretrain_cmt.__file__).startswith(src), pretrain_cmt.__file__

    def build_projector():      # pretrain_cmt.py:19-32 with the host as device
        D = pretrain_cmt.BEV_DIM
        projector = bev_utils.PointCloud(math.radians(90), 1, feature_map_height=14, feature_map_width=14, map_dim=D,
                                         map_res=pretrain_cmt.BEV_RES, world_shift_origin=torch.zeros(3),
                                         z_clip_threshold=0.5, device=torch.device("cpu"))
        return projector, bev_utils.bevpos_polar(D).reshape(D * D, 3)[None, :, :]

    pretrain_cmt.build_projector = build_projector
    return pretrain_cmt


def main():
    from bevbert_b200.model.ce_pretrain import GlocalTextPathCMTPreTraining
    cfg, scfg = case()
    ours = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=WEIGHT_SEED)
    sd = {k: v.detach().clone() for k, v in ours.state_dict().items()}
    pretrain_cmt = load_ce_modules()
    ref = pretrain_cmt.GlocalTextPathCMTPreTraining(cfg)
    missing, unexpected = ref.load_state_dict(sd, strict=False)
    assert not [k for k in missing if not k.endswith("decoder.weight")] and not unexpected, (missing, unexpected)
    ref.tie_weights()
    ref.train()
    for m in ref.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
        if isinstance(m, torch.nn.MultiheadAttention):
            m.dropout = 0.0
    gold = {"shapes": {k: tuple(v.shape) for k, v in ref.state_dict().items()},
            "param_order": [n for n, _ in ref.named_parameters()], "weight_seed": WEIGHT_SEED,
            "batch_seed": BATCH_SEED, "tasks": {}}
    for task in TASKS:
        b = synth.make_batch(scfg, seed=BATCH_SEED, task=task)
        ref.zero_grad()
        loss = ref(synth.clone_batch(b), task, compute_loss=True)
        loss.mean().backward()
        with torch.no_grad():
            logits = ref(synth.clone_batch(b), task, compute_loss=False)
        logits = logits if isinstance(logits, tuple) else (logits,)
        grads = {n: p.grad.detach() for n, p in ref.named_parameters() if p.grad is not None}
        gold["tasks"][task] = {
            "loss": loss.detach().clone(),
            "logits": [t.detach().clone() for t in logits[:3]],
            "grad_norms": {n: float(g.norm()) for n, g in grads.items()},
            "grad_proj": {n: grad_projections(n, g) for n, g in grads.items()},
            "grads": {n: grads[n].clone() for n in FULL_GRADS if n in grads},
        }
        print(task, "loss mean %.6f" % float(loss.mean()), "n_grads", len(grads))
    torch.save(gold, os.path.join(os.path.dirname(os.path.abspath(__file__)), "small_ce.pt"))


if __name__ == "__main__":
    main()
