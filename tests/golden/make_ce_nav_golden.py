"""Generates tests/golden/small_ce_nav.pt by running the UNMODIFIED VLN-CE navigation network
(bevbert_ce/vlnce_baselines/models/bev/vilmodel_cmt.py of the reference checkout located by oracle/ref_shim.py, env
BEVBERT_REFERENCE) and the CE trainer's BEV helpers (graph_utils.GraphMap.gather_node_pc, bev_utils.transfrom3D,
bev_utils.PointCloud.project_bev) on seeded weights and inputs:

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_ce_nav_golden.py

`vlnce_baselines/__init__.py` imports habitat and every trainer, so the modules are imported through stub parent
packages whose `__path__` points at the reference directories and whose own `__init__` never runs.  The habitat,
matplotlib and torch_scatter imports of graph_utils.py / bev_utils.py are stubbed (the stubs are not called on the
pinned paths, except scatter_mean, restated as in oracle/ref_shim.py); transformers' init hook is the ref_shim one.

Stored (data only), for each (use_depth_embedding, graph_sprels) of tests/ce_nav_cases.VARIANTS: the outputs of the
three calls at B = 3 (embeddings by their first channels and row norms); a teacher-forced rollout's loss, every parameter gradient's norm and its projections on the
seeded directions of make_ce_golden.grad_probes; the state_dict key -> shape map and the parameter order; and the keys
the reference's from_pretrained loads from a CE pre-training state_dict remapped as get_vlnbert_models remaps it.
BEV: gather_node_pc's node order on a small graph, transfrom3D of a few headings, and project_bev of a seeded cloud."""
import importlib
import math
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.dirname(os.path.abspath(__file__))]

import ce_nav_cases as C  # noqa: E402
from bevbert_b200 import synth  # noqa: E402
from oracle import ref_shim  # noqa: E402

B = 3


def _pkg(name, path):
    m = types.ModuleType(name)
    m.__path__ = [path]
    sys.modules[name] = m
    return m


def load_ce_modules():
    """-> (vilmodel_cmt, graph_utils, bev_utils) of the reference CE tree"""
    base = os.path.join(ref_shim.REF_ROOT, "bevbert_ce", "vlnce_baselines")
    if not os.path.isdir(base):
        raise RuntimeError("CE reference tree not found under %s" % ref_shim.REF_ROOT)
    sys.dont_write_bytecode = True
    _pkg("vlnce_baselines", base)
    _pkg("vlnce_baselines.common", os.path.join(base, "common"))
    _pkg("vlnce_baselines.models", os.path.join(base, "models"))
    _pkg("vlnce_baselines.models.bev", os.path.join(base, "models", "bev"))

    def unused(*a, **k):
        raise NotImplementedError("habitat stub")
    for name, attrs in (("habitat", {}), ("habitat.tasks", {}), ("habitat.tasks.utils", {"cartesian_to_polar": unused}),
                        ("habitat.utils", {}), ("habitat.utils.geometry_utils",
                                                {"quaternion_rotate_vector": unused, "quaternion_from_coeff": unused}),
                        ("matplotlib", {}), ("matplotlib.pyplot", {})):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__dict__.update(attrs)
            sys.modules[name] = m
    if "torch_scatter" not in sys.modules:
        stub = types.ModuleType("torch_scatter")
        stub.scatter_mean = ref_shim._scatter_mean
        stub.scatter_max = unused
        sys.modules["torch_scatter"] = stub
    vil = importlib.import_module("vlnce_baselines.models.bev.vilmodel_cmt")
    vil.BertPreTrainedModel.init_weights = lambda self: None
    vil.BertPreTrainedModel.all_tied_weights_keys = {}     # transformers 5.x asks every model for its tied weights
    graph_utils = importlib.import_module("vlnce_baselines.models.graph_utils")
    bev_utils = importlib.import_module("vlnce_baselines.models.bev_utils")
    for m in (vil, graph_utils, bev_utils):
        assert m.__file__.startswith(base), m.__file__
    return vil, graph_utils, bev_utils


def _detach(x):
    if isinstance(x, dict):
        return {k: _detach(v) for k, v in x.items()}
    if isinstance(x, (tuple, list)):
        return type(x)(_detach(v) for v in x)
    return x.detach().clone() if torch.is_tensor(x) else x


def calls(net, B):
    """the three calls once, on step-0 inputs, with gradients off -> {"txt", "pano", "nav"}; embeddings as
    C.embed_pin (first channels and row norms), masks and logits in full"""
    with torch.no_grad():
        _, outs = C.rollout(net, B, steps=1)
    o = _detach(outs[0])
    nav = dict(o["nav"], gmap_embeds=C.embed_pin(o["nav"]["gmap_embeds"]))
    return {"txt": C.embed_pin(o["txt"]), "pano": (C.embed_pin(o["pano"][0]), o["pano"][1]), "nav": nav}


def pretrain_remap(sd):
    """vlnbert_init.py:21-30: head keys get `bert.` put in front"""
    return {("bert." + k if ("_head" in k or "sap_fuse" in k) else k): v for k, v in sd.items()}


def project_feats(n):
    return synth.det_uniform((2, n, 768), 21, 4, -2.0, 2.0)


def bev_cases(graph_utils, bev_utils):
    import networkx as nx
    out = {}
    # gather_node_pc on a path graph a - b - c - d with a branch b - e: node order and orders 0, 1, 2
    gm = graph_utils.GraphMap.__new__(graph_utils.GraphMap)
    g = nx.Graph()
    g.add_weighted_edges_from([("a", "b", 1.0), ("b", "c", 1.0), ("c", "d", 1.0), ("b", "e", 2.0)])
    gm.shortest_path = dict(nx.all_pairs_dijkstra_path(g))
    gm.node_pc = {}
    for k, vp in enumerate(["c", "a", "e", "b", "d"]):
        gm.update_node_pc(vp, torch.full((k + 1, 3), float(k)), torch.zeros(k + 1, dtype=torch.bool),
                          torch.full((k + 1, 2), float(k)))
    out["gather"] = {(vp, order): gm.gather_node_pc(vp, order)[0][:, 0].tolist() for vp in "abcde" for order in (0, 1, 2)}
    # transfrom3D at the headings the splat uses (-heading, elevation 0)
    hd = np.array([0.0, 0.3, -1.2, math.pi / 2, -math.pi, 2.5, 3 * math.pi / 2 - 1e-3])
    xyzhe = np.zeros((len(hd), 5))
    xyzhe[:, 3] = hd
    out["headings"] = torch.from_numpy(hd)
    out["T"] = torch.from_numpy(bev_utils.transfrom3D(xyzhe))
    # project_bev at 11 x 11 / 1 m of an ego-frame cloud: in-map, outside, above the clip, no-depth and boundary points
    proj = bev_utils.PointCloud(math.radians(90), 1, feature_map_height=14, feature_map_width=14, map_dim=11, map_res=1,
                                world_shift_origin=torch.zeros(3), z_clip_threshold=0.5, device=torch.device("cpu"))
    n = 600
    pc = synth.det_uniform((2, n, 3), 21, 1, -7.0, 7.0)
    pc[:, :, 1] = synth.det_uniform((2, n), 21, 2, -1.0, 0.8)
    pc[0, :8] = torch.tensor([[0.5, 0, 0], [-0.5, 0, 0], [5.5, 0, 5.5], [-5.5, 0, -5.5], [5.51, 0, 0], [0, 0.5, 0],
                              [0, 0.50001, 0], [1.5, 0, -2.5]])
    nod = synth.det_uniform((2, n), 21, 3) < 0.1
    feat = project_feats(n)
    bev, ob = proj.project_bev(pc, nod, feat)
    # the cell means of the first 8 channels pin every point's cell (channels are pooled independently)
    out["project"] = {"pc": pc, "no_depth": nod, "bev8": bev.reshape(2, 121, 768)[..., :8].clone(),
                      "ob": ob.reshape(2, 121)}
    return out


def main():
    from bevbert_b200.model.ce_nav import GlocalTextPathNavCMT
    from bevbert_b200.model.ce_pretrain import GlocalTextPathCMTPreTraining
    from bevbert_b200.config import make_ce_config
    from make_ce_golden import grad_projections
    vil, graph_utils, bev_utils = load_ce_modules()
    gold = {"weight_seed": C.WEIGHT_SEED, "B": B, "variants": {}}
    for depth, sprels in C.VARIANTS:
        cfg = C.config(depth, sprels)
        sd = synth.det_init_(GlocalTextPathNavCMT(cfg), seed=C.WEIGHT_SEED).state_dict()
        ref = vil.GlocalTextPathNavCMT(cfg)
        missing, unexpected = ref.load_state_dict(sd, strict=True)
        ref.eval()
        v = {"shapes": {k: tuple(t.shape) for k, t in ref.state_dict().items()},
             "param_order": [n for n, _ in ref.named_parameters()], "calls": calls(ref, B)}
        ref.train()
        for m in ref.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
            if isinstance(m, torch.nn.MultiheadAttention):
                m.dropout = 0.0
        ref.zero_grad()
        loss, _ = C.rollout(ref, B)
        loss.backward()
        grads = {n: p.grad.detach() for n, p in ref.named_parameters() if p.grad is not None}
        v["loss"] = float(loss.detach())
        v["grad_norms"] = {n: float(g.norm()) for n, g in grads.items()}
        v["grad_proj"] = {n: grad_projections(n, g) for n, g in grads.items()}
        gold["variants"][(depth, sprels)] = v
        print("depth", depth, "sprels", sprels, "loss %.6f" % float(loss), "n_grads", len(grads))
    # the keys from_pretrained loads from a CE pre-training checkpoint, remapped by get_vlnbert_models
    pt = GlocalTextPathCMTPreTraining(make_ce_config(small=True))
    remapped = pretrain_remap(pt.state_dict())
    cfg = C.config(True, True)
    before = {k: t.clone() for k, t in vil.GlocalTextPathNavCMT(cfg).state_dict().items()}
    for t in remapped.values():
        t.fill_(0.5) if t.is_floating_point() else None
    ref = vil.GlocalTextPathNavCMT.from_pretrained(None, config=cfg, state_dict=remapped)
    loaded = sorted(k for k, t in ref.state_dict().items() if t.is_floating_point() and bool((t == 0.5).all()))
    gold["pretrain_loaded"] = loaded
    gold["pretrain_keys"] = sorted(remapped)
    print("from_pretrained loads", len(loaded), "of", len(before), "keys")
    gold["bev"] = bev_cases(graph_utils, bev_utils)
    torch.save(gold, os.path.join(os.path.dirname(os.path.abspath(__file__)), "small_ce_nav.pt"))


if __name__ == "__main__":
    main()
