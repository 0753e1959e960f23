"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the VLN-CE trainer's `lift` (ss_trainer_BEV.py:386-410), the oracle
of bb_bev_lift_points / agent_bev.ce_lift.  Paths are relative to bevbert_ce/vlnce_baselines of the reference.

The trainer module cannot be imported (habitat_baselines, lmdb, gym, the simulator).  `lift` builds its heading fan
with transfrom3D, then calls PointCloud.forward (models/bev_utils.py:349-378) on depth_grid * 10: point_cloud's
camera-frame xyz1 (:139-172), bmm with T (:198), minus world_shift_origin (:243), and the no-depth mask (:371).
Everything but the bmm is restated with the reference's own expressions; the camera-to-world product is written as
each row of T dotted with (x, y, z, 1) left to right in fp32 (the reference leaves that order to bmm).  The pieces are
pinned to the unmodified reference by tests/golden/small_ce_lift.pt."""
import math

import numpy as np
import torch

from ce_nav_bev_oracle import transfrom3D

VIEWS, GRID = 12, 14


def lift_T(cur_pos, headings):
    """lift's fan (:391-400): (B*12, 4, 4) float32.  headings[i] = heading_from_quaternion(cur_ori[i])"""
    xyzhe = np.zeros([len(cur_pos), VIEWS, 5])
    for i, (pos_i, h) in enumerate(zip(cur_pos, headings)):
        x, y, z = pos_i
        xyzhe[i, :, 0] = x
        xyzhe[i, :, 1] = y
        xyzhe[i, :, 2] = z
        xyzhe[i, :, 3] = -np.arange(12) * np.radians(30) + h
        xyzhe[i, :, 4] = np.pi
    return torch.from_numpy(transfrom3D(xyzhe.reshape(-1, 5)))


def intrinsics(vfov=math.radians(90), fmh=GRID, fmw=GRID):
    """compute_intrinsic_matrix (:91-100): fx, fy, cx, cy as float32 tensors"""
    hfov = fmw / fmh * vfov
    K = torch.Tensor([[fmw / (2.0 * math.tan(hfov / 2.0)), 0, fmw / 2.0],
                      [0, fmh / (2.0 * math.tan(vfov / 2.0)), fmh / 2.0], [0, 0, 1.0]])
    return K[0, 0], K[1, 1], K[0, 2], K[1, 2]


def camera_xyz1(depth_grid, vfov=math.radians(90)):
    """depth_grid * 10 (:402) through point_cloud (:115-131, 167-172): -> xyz1 (N, 196, 4) float32, mask (N, 196)"""
    depth = depth_grid.reshape(-1, GRID, GRID) * 10
    N = depth.shape[0]
    fx, fy, cx, cy = intrinsics(vfov)
    x_rows = torch.arange(GRID).unsqueeze(0).repeat((GRID, 1)).unsqueeze(0).repeat((N, 1, 1)).float()
    y_cols = torch.arange(GRID).unsqueeze(1).repeat((1, GRID)).unsqueeze(0).repeat((N, 1, 1)).float()
    x_scale = (x_rows + 0.5 - cx) / fx
    y_scale = (y_cols + 0.5 - cy) / fy
    z = depth / float(1.0)
    xyz1 = torch.stack([z * x_scale, z * y_scale, z, torch.ones_like(z)], -1)
    return xyz1.reshape(N, GRID * GRID, 4), (depth == 0).reshape(N, GRID * GRID)


def world_points(xyz1, T, shift):
    """T * xyz1 with each row of T dotted left to right in fp32, minus shift: (N, P, 4), (N, 4, 4), (3,) -> (N, P, 3)"""
    x, y, z = xyz1[..., 0], xyz1[..., 1], xyz1[..., 2]
    rows = []
    for j in range(3):
        t = T[:, j, :, None]
        rows.append((((t[:, 0] * x + t[:, 1] * y) + t[:, 2] * z) + t[:, 3]) - shift[j])
    return torch.stack(rows, -1)


def lift(cur_pos, headings, depth_grid, shift=torch.zeros(3), vfov=math.radians(90)):
    """-> {T (B*12,4,4), xyz1 (B*12,196,4), pc (B,2352,3), pc_mask (B,2352)}, float32 / bool, on the CPU"""
    B = len(cur_pos)
    T = lift_T(cur_pos, headings)
    xyz1, mask = camera_xyz1(depth_grid.cpu(), vfov)
    pc = world_points(xyz1, T, shift.cpu())
    return {"T": T, "xyz1": xyz1, "pc": pc.reshape(B, -1, 3), "pc_mask": mask.reshape(B, -1)}
