"""Generates tests/golden/small_ce_lift.pt by running the VLN-CE trainer's own `lift` (ss_trainer_BEV.py:386-410)
over the UNMODIFIED PointCloud and transfrom3D (models/bev_utils.py) and graph_utils.heading_from_quaternion of the
reference checkout located by oracle/ref_shim.py (env BEVBERT_REFERENCE), on the seeded cases of
tests/ce_lift_cases.py, on the CPU:

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_ce_lift_golden.py

The modules are imported through the stub parent packages of make_ce_gmap_golden.py; habitat's quaternion helpers are
ce_lift_cases' restatements, matplotlib is a stub and torch_scatter is oracle/ref_shim.py's (neither is called here).
ss_trainer_BEV.py cannot be imported, so only the source of `lift` is taken from it (by its syntax tree) and run with
the module's own names for what it uses; its `.cuda()` calls return the CPU tensor.  Per case it stores the input
digests, the headings, the matrices T bmm receives, the camera-frame xyz1 of point_cloud, the no-depth mask and the
world points.  xyz1 is stored as its SHA-256 and shape (it is 4/3 the size of the points)."""
import ast
import importlib
import math
import os
import sys
import textwrap
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.dirname(os.path.abspath(__file__))]

import ce_lift_cases as C  # noqa: E402
import make_ce_gmap_golden as G  # noqa: E402
from oracle import ref_shim  # noqa: E402


def load():
    """-> (graph_utils, bev_utils, the trainer's lift as a function of (self, cur_pos, cur_ori, rgb_grid, depth_grid))"""
    base = os.path.join(ref_shim.REF_ROOT, "bevbert_ce", "vlnce_baselines")
    if not os.path.isdir(base):
        raise RuntimeError("CE reference tree not found under %s" % ref_shim.REF_ROOT)
    sys.dont_write_bytecode = True
    G._pkg("vlnce_baselines", base)
    G._pkg("vlnce_baselines.models", os.path.join(base, "models"))
    sys.modules.update(C.habitat_stubs())
    for name in ("matplotlib", "matplotlib.pyplot"):
        sys.modules.setdefault(name, types.ModuleType(name))
    scatter = types.ModuleType("torch_scatter")
    scatter.scatter_mean = ref_shim._scatter_mean
    scatter.scatter_max = None
    sys.modules.setdefault("torch_scatter", scatter)
    gu = importlib.import_module("vlnce_baselines.models.graph_utils")
    bu = importlib.import_module("vlnce_baselines.models.bev_utils")
    assert gu.__file__.startswith(base) and bu.__file__.startswith(base)
    src = open(os.path.join(base, "ss_trainer_BEV.py")).read()
    fn = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == "lift")
    ns = {"torch": torch, "np": np, "transfrom3D": bu.transfrom3D, "heading_from_quaternion": gu.heading_from_quaternion}
    exec(compile(textwrap.dedent(ast.get_source_segment(src, fn)), "ss_trainer_BEV.py", "exec"), ns)
    return gu, bu, ns["lift"]


def run(bu, lift, case):
    """the trainer's lift on one case, recording what PointCloud.forward hands to point_cloud and bmm"""
    cur_pos, cur_ori, depth, shift, digests = C.case_inputs(case)
    B = case["B"]
    trainer = types.SimpleNamespace(envs=types.SimpleNamespace(num_envs=B))
    trainer.projector = bu.PointCloud(math.radians(90), 1, feature_map_height=14, feature_map_width=14, map_dim=11,
                                      map_res=1, world_shift_origin=shift.clone(), z_clip_threshold=0.5, device="cpu")
    seen = {}
    point_cloud, to_world = trainer.projector.point_cloud, trainer.projector.transform_camera_to_world

    def rec_point_cloud(*a, **k):
        seen["xyz1"] = point_cloud(*a, **k)
        return seen["xyz1"]

    def rec_to_world(xyz1, T):
        seen["T"] = T
        return to_world(xyz1, T)
    trainer.projector.point_cloud, trainer.projector.transform_camera_to_world = rec_point_cloud, rec_to_world
    rgb = C.rgb_grid(B, "cpu")
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda t, *a, **k: t
    try:
        pc, mask, feat = lift(trainer, cur_pos, cur_ori, rgb, depth)
    finally:
        torch.Tensor.cuda = cuda
    assert feat.data_ptr() == rgb.data_ptr() and feat.shape == (B, 2352, 768)
    assert pc.dtype == torch.float32 and mask.dtype == torch.bool and seen["T"].dtype == torch.float32
    xyz1 = seen["xyz1"].reshape(B * 12, 196, 4).contiguous()
    return {"case": case, "input_digests": digests, "T": seen["T"].clone(), "xyz1_digest": C.sha(xyz1.numpy()),
            "xyz1_shape": tuple(xyz1.shape), "pc_mask": mask.clone(), "pc": pc.clone()}


def main():
    gu, bu, lift = load()
    gold = {"cases": []}
    for case in C.CASES:
        cur_pos, cur_ori, _, _, _ = C.case_inputs(case)
        out = run(bu, lift, case)
        out["headings"] = [float(gu.heading_from_quaternion(o)) for o in cur_ori]
        print("case %d: B=%d, %d no-depth points" % (case["seed"], case["B"], int(out["pc_mask"].sum())))
        gold["cases"].append(out)
    torch.save(gold, os.path.join(os.path.dirname(os.path.abspath(__file__)), "small_ce_lift.pt"))


if __name__ == "__main__":
    main()
