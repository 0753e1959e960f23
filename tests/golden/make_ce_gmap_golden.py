"""Generates tests/golden/small_ce_gmap.pt by running the UNMODIFIED VLN-CE GraphMap (bevbert_ce/vlnce_baselines/
models/graph_utils.py: update_graph, delete_ghost, get_node_embeds, get_pos_fts, front_to_ghost_dist) and the trainer's
`_nav_gmap_variable` (ss_trainer_BEV.py:534-611) of the reference checkout located by oracle/ref_shim.py (env
BEVBERT_REFERENCE) on seeded episodes (tests/ce_gmap_cases.GOLDEN_CASES), on the CPU:

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_ce_gmap_golden.py

graph_utils.py and common/ops.py are imported through stub parent packages (`vlnce_baselines/__init__.py` imports
habitat and every trainer); their habitat and matplotlib imports are stubs, and `heading_from_quaternion` reads the
episode's heading directly.  ss_trainer_BEV.py imports habitat, lmdb and the simulator extensions, so only the source of
`_nav_gmap_variable` is taken from it (by its syntax tree) and run with the module's own names for what it uses; its
`.cuda()` calls return the CPU tensor.  Each episode runs twice, from the same seeds:
  * with the rollout's embeddings (ss_trainer_BEV.py:1032-1033, 1060-1066): per step the digest and shape of
    gmap_img_fts, gmap_vp_ids and no_vp_left;
  * with the host half of graphs.install_ce_gmap_features on the same classes (bevbert_b200.ce_gmap.attach and
    trainer_method): per step the handles the method's get_node_embeds calls gave, as labels.
Inputs are not stored: tests regenerate them from the seeds and check the stored SHA-256 digests."""
import ast
import hashlib
import importlib
import os
import sys
import textwrap
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.dirname(os.path.abspath(__file__))]

import ce_gmap_cases as C  # noqa: E402
from oracle import ref_shim  # noqa: E402


def digest(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def _pkg(name, path):
    m = types.ModuleType(name)
    m.__path__ = [path]
    sys.modules[name] = m


def load():
    """-> (graph_utils module, the trainer's _nav_gmap_variable as a function of (self, cur_vp, cur_pos, cur_ori))"""
    base = os.path.join(ref_shim.REF_ROOT, "bevbert_ce", "vlnce_baselines")
    if not os.path.isdir(base):
        raise RuntimeError("CE reference tree not found under %s" % ref_shim.REF_ROOT)
    sys.dont_write_bytecode = True
    _pkg("vlnce_baselines", base)
    _pkg("vlnce_baselines.common", os.path.join(base, "common"))
    _pkg("vlnce_baselines.models", os.path.join(base, "models"))

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
    gu = importlib.import_module("vlnce_baselines.models.graph_utils")
    ops = importlib.import_module("vlnce_baselines.common.ops")
    assert gu.__file__.startswith(base) and ops.__file__.startswith(base)
    gu.heading_from_quaternion = float          # the episodes give each orientation as its heading
    src = open(os.path.join(base, "ss_trainer_BEV.py")).read()
    fn = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == "_nav_gmap_variable")
    ns = {"torch": torch, "np": np, "pad_sequence": torch.nn.utils.rnn.pad_sequence, "MAX_DIST": gu.MAX_DIST,
          "pad_tensors_wgrad": ops.pad_tensors_wgrad, "gen_seq_masks": ops.gen_seq_masks}
    exec(compile(textwrap.dedent(ast.get_source_segment(src, fn)), "ss_trainer_BEV.py", "exec"), ns)
    return gu, ns["_nav_gmap_variable"]


class Trainer:
    """what _nav_gmap_variable reads of the trainer: gmaps and envs.num_envs"""

    def __init__(self, method):
        self.envs = types.SimpleNamespace()
        self._method = method

    def __call__(self, cur_vp, cur_pos, cur_ori):
        self.envs.num_envs = len(self.gmaps)
        cuda = torch.Tensor.cuda
        torch.Tensor.cuda = lambda t, *a, **k: t
        try:
            return self._method(self, cur_vp, cur_pos, cur_ori)
        finally:
            torch.Tensor.cuda = cuda


def main():
    gu, method = load()
    gold = {"cases": []}
    for case in C.GOLDEN_CASES:
        t = Trainer(method)
        ref = C.golden_episode(case, gu.GraphMap, t, t)
        t = Trainer(method)
        ins = C.golden_episode(case, gu.GraphMap, t, t, handles=True)
        steps = []
        for (out, _, dg), (out_h, rows, dg_h) in zip(ref, ins):
            assert dg == dg_h and out["gmap_vp_ids"] == out_h["gmap_vp_ids"]
            f = out["gmap_img_fts"]
            assert f.dtype == torch.float32
            steps.append({"input_digests": dg, "fts_digest": digest(f), "fts_shape": tuple(f.shape),
                          "gmap_vp_ids": out["gmap_vp_ids"], "no_vp_left": out["no_vp_left"], "rows": rows})
        ghosts = sum(len(r) > 1 for s in steps for row in s["rows"] for r in row if r[0] != "n")
        print("case %d: %d steps, %d merged-ghost rows" % (case["seed"], len(steps), ghosts))
        gold["cases"].append({"case": case, "steps": steps})
    torch.save(gold, os.path.join(os.path.dirname(os.path.abspath(__file__)), "small_ce_gmap.pt"))


if __name__ == "__main__":
    main()
