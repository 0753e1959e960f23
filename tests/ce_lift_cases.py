"""Seeded inputs of the VLN-CE trainer's `lift` (ss_trainer_BEV.py:386-410), shared by the golden generator
(tests/golden/make_ce_lift_golden.py, which runs the unmodified `lift`, PointCloud and transfrom3D), the CPU tests and
the GPU tests of agent_bev.ce_lift / bb_bev_lift_points.

Orientations are habitat quaternions, coefficients [x, y, z, w], about the vertical (y) axis.  The habitat functions
graph_utils.heading_from_quaternion calls (quaternion_from_coeff, quaternion_rotate_vector, cartesian_to_polar) are
restated below from habitat-lab's public API, so that the reference's function runs unmodified on top of them;
`heading_from_quaternion` is that function over them, the one the stand-in trainer's module gives ce_lift."""
import hashlib
import math
import types

import numpy as np
import torch

from ce_nav_bev_cases import StubTrainer

CASES = [
    {"seed": 61, "B": 1, "shift": (0.0, 0.0, 0.0)},
    {"seed": 62, "B": 3, "shift": (0.25, -1.5, 3.0)},       # the kernel subtracts any world_shift_origin
    {"seed": 63, "B": 8, "shift": (0.0, 0.0, 0.0)},
]


class Quaternion:
    """the part of numpy-quaternion's quaternion that habitat's helpers use"""

    def __init__(self, w, x, y, z):
        self.w, self.x, self.y, self.z = float(w), float(x), float(y), float(z)

    def __mul__(self, o):
        return Quaternion(self.w * o.w - self.x * o.x - self.y * o.y - self.z * o.z,
                          self.w * o.x + self.x * o.w + self.y * o.z - self.z * o.y,
                          self.w * o.y - self.x * o.z + self.y * o.w + self.z * o.x,
                          self.w * o.z + self.x * o.y - self.y * o.x + self.z * o.w)

    def inverse(self):
        n = self.w * self.w + self.x * self.x + self.y * self.y + self.z * self.z
        return Quaternion(self.w / n, -self.x / n, -self.y / n, -self.z / n)

    @property
    def imag(self):
        return np.array([self.x, self.y, self.z])


def quaternion_from_coeff(coeffs):
    """habitat.utils.geometry_utils.quaternion_from_coeff: [x, y, z, w] -> quaternion"""
    return Quaternion(coeffs[3], coeffs[0], coeffs[1], coeffs[2])


def quaternion_rotate_vector(quat, v):
    """habitat.utils.geometry_utils.quaternion_rotate_vector: quat * (0, v) * quat^-1, imaginary part"""
    return (quat * Quaternion(0.0, *v) * quat.inverse()).imag


def cartesian_to_polar(x, y):
    """habitat.tasks.utils.cartesian_to_polar"""
    return np.sqrt(x ** 2 + y ** 2), np.arctan2(y, x)


def heading_from_quaternion(quat):
    """graph_utils.heading_from_quaternion (graph_utils.py:58-63) over the helpers above"""
    q = quaternion_from_coeff(quat)
    heading_vector = quaternion_rotate_vector(q.inverse(), np.array([0, 0, -1]))
    phi = cartesian_to_polar(-heading_vector[2], heading_vector[0])[1]
    return phi % (2 * np.pi)


def habitat_stubs():
    """{module name: module} of the habitat helpers above, for importing the reference's graph_utils"""
    mods = {}
    for name, attrs in (("habitat", {}), ("habitat.tasks", {}),
                        ("habitat.tasks.utils", {"cartesian_to_polar": cartesian_to_polar}), ("habitat.utils", {}),
                        ("habitat.utils.geometry_utils", {"quaternion_rotate_vector": quaternion_rotate_vector,
                                                          "quaternion_from_coeff": quaternion_from_coeff})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        mods[name] = m
    return mods


def quaternion_at(theta):
    """habitat coefficients [x, y, z, w] of a rotation by theta about +y"""
    return np.array([0.0, math.sin(theta / 2), 0.0, math.cos(theta / 2)])


def depth_grid(rng, B):
    """(B, 12, 196, 1) float32 like the waypoint step's pano_depth_grid (means of depths in [0, 1]), with exact zeros,
    subnormal values, the smallest normal, values at 1 and every pixel of one view without depth"""
    d = rng.random((B, 12, 196, 1), dtype=np.float32)
    flat = d.reshape(-1)
    n = flat.size
    pick = rng.permutation(n)
    k = max(n // 10, 8)
    flat[pick[:k]] = 0.0
    flat[pick[k:k + 8]] = np.array([1e-45, 3e-45, 1e-42, 1e-40, 1e-39, 1.1754942e-38, 1.1754944e-38, 1.0], np.float32)
    d[0, 5] = 0.0
    return torch.from_numpy(d)


def case_inputs(case):
    """-> (cur_pos (list of (3,) float64), cur_ori (list of quaternions), depth_grid (B,12,196,1) float32,
    world_shift (3,) float32, digests {name: sha256})"""
    rng = np.random.default_rng(case["seed"])
    B = case["B"]
    cur_pos = [rng.uniform(-50, 50, 3) for _ in range(B)]
    fixed = [0.0, math.pi / 2, math.pi, 3 * math.pi / 2, -0.3]
    thetas = [fixed[i] if i < len(fixed) and B > 1 else float(rng.uniform(-math.pi, math.pi)) for i in range(B)]
    cur_ori = [quaternion_at(t) for t in thetas]
    d = depth_grid(rng, B)
    shift = torch.tensor(case["shift"], dtype=torch.float32)
    digests = {"cur_pos": sha(np.stack(cur_pos)), "cur_ori": sha(np.stack(cur_ori)), "depth_grid": sha(d.numpy()),
               "shift": sha(shift.numpy())}
    return cur_pos, cur_ori, d, shift, digests


def rgb_grid(B, device, seed=0):
    """(B, 12, 196, 768) float32 features (their values only travel through as the cloud's features)"""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 12, 196, 768, generator=g).to(device)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class Projector:
    """what lift reads of the trainer's PointCloud (ss_trainer_BEV.py:204-215)"""

    def __init__(self, device, shift=(0.0, 0.0, 0.0), vfov=math.radians(90), fmh=14, fmw=14):
        self.vfov, self.fmh, self.fmw = vfov, fmh, fmw
        self.world_shift_origin = torch.tensor(shift, dtype=torch.float32, device=device)


class LiftTrainer(StubTrainer):
    """ce_nav_bev_cases' stand-in trainer with lift's projector; this module's heading_from_quaternion is the one
    ce_lift and ce_nav_bev_variable take for it"""

    def __init__(self, B, device, shift=(0.0, 0.0, 0.0)):
        super().__init__(B, device)
        self.projector = Projector(device, shift)
