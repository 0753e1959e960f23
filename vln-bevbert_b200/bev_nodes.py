"""Tensor-level wrappers of the node point-cloud kernels (include/bevbert_b200.h): `bb_bev_splat_nodes`, the agents'
per-step BEV pooled straight from the navigation graph's node clouds, and `bb_bev_lift_points`, which makes the VLN-CE
trainer's node clouds.  The splat wrapper keeps host state (the pinned launch tables), which is why it lives beside
`kernels.py` rather than in it; the lift wrapper sits with it because it produces the clouds the splat reads.  Every
wrapper only checks arguments, fills a table where there is one and launches, and raises without the CUDA library."""
import numpy as np
import torch

from . import _lib
from .kernels import BF16, _capturing, _req, _stream


class _NodeTableSlot:
    """Pinned host rows + device copy of one `bb_bev_splat_nodes` launch table.  The library copies the pinned rows
    asynchronously; `busy` is an event behind the launch that read them, and the host waits on it before it rewrites
    the rows (the same guard as `MtTable`)."""

    def __init__(self):
        self.host = self.dev = self.busy = None

    def acquire(self, nbytes, device):
        if self.busy is not None:
            self.busy.synchronize()
            self.busy = None
        if self.host is None or self.host.numel() < nbytes or self.dev.device != device:
            n = max(1024, 1 << (nbytes - 1).bit_length())
            self.host = torch.empty(n, dtype=torch.uint8).pin_memory()
            self.dev = torch.empty(n, dtype=torch.uint8, device=device)
        return self.host, self.dev

    def mark_busy(self):
        self.busy = torch.cuda.Event()
        self.busy.record()


_NODE_SLOTS = [_NodeTableSlot(), _NodeTableSlot()]   # alternated, so the host can build one call ahead of the device
_NODE_TURN = [0]


def bev_splat_nodes(clouds, S_w2c, T_w2c, map_dim, map_res, y_clip=0.5, C=None):
    """Agent-side BEV from node point clouds (bb_bev_splat_nodes).  clouds: a list over samples of lists of
    (pc f32 (n,3) world frame, no_depth bool/uint8 (n,), feat f32 | bf16 (n,C)) node tuples, all contiguous on the
    device of S_w2c (B,3) / T_w2c (B,4,4) f32; a node may appear in several samples.  C is only needed when no sample
    has a node.  -> (bev f32 (B, map_dim**2, C), ob_mask bool (B, map_dim**2))."""
    lib = _lib.load()
    _req(S_w2c, torch.float32, "S_w2c")
    _req(T_w2c, torch.float32, "T_w2c")
    if _capturing():
        raise RuntimeError("bev_splat_nodes builds its launch table on the host at every call and cannot be captured")
    B = len(clouds)
    dev = S_w2c.device
    if T_w2c.device != dev:
        raise RuntimeError("S_w2c and T_w2c must be on the same device")
    if tuple(S_w2c.shape) != (B, 3) or tuple(T_w2c.shape) != (B, 4, 4):
        raise ValueError("S_w2c must be (B, 3) and T_w2c (B, 4, 4) for B = %d samples, got %s and %s"
                         % (B, tuple(S_w2c.shape), tuple(T_w2c.shape)))
    rows, offs, fdt = [], [0], None
    for b, nodes in enumerate(clouds):
        for j, node in enumerate(nodes):
            pc, nod, ft = node
            where = "clouds[%d][%d]" % (b, j)
            for t, what in ((pc, "points"), (nod, "no-depth mask"), (ft, "features")):
                if not t.is_cuda or t.device != dev:
                    raise RuntimeError("%s: %s must be a CUDA tensor on %s, got %s" % (where, what, dev, t.device))
                if not t.is_contiguous():
                    raise ValueError("%s: %s must be contiguous" % (where, what))
            if pc.dtype != torch.float32:
                raise TypeError("%s: points must be torch.float32, got %s" % (where, pc.dtype))
            if nod.dtype not in (torch.bool, torch.uint8):
                raise TypeError("%s: no-depth mask must be bool or uint8, got %s" % (where, nod.dtype))
            if ft.dtype not in (torch.float32, BF16) or (fdt is not None and ft.dtype != fdt):
                raise TypeError("%s: features must be float32 or bfloat16 like the other nodes, got %s" % (where, ft.dtype))
            fdt = ft.dtype
            n = pc.shape[0]
            if pc.dim() != 2 or pc.shape[1] != 3 or tuple(nod.shape) != (n,) or ft.dim() != 2 or ft.shape[0] != n:
                raise ValueError("%s: expected points (n,3), mask (n,), features (n,C); got %s, %s, %s"
                                 % (where, tuple(pc.shape), tuple(nod.shape), tuple(ft.shape)))
            if C is None:
                C = ft.shape[1]
            elif ft.shape[1] != C:
                raise ValueError("%s: %d feature columns, expected %d" % (where, ft.shape[1], C))
            rows.append((pc.data_ptr(), nod.data_ptr(), ft.data_ptr(), n))
        offs.append(len(rows))
    if C is None:
        raise ValueError("bev_splat_nodes: no sample has a node; pass C")
    ncell = map_dim * map_dim
    bev = torch.empty(B, ncell, C, dtype=torch.float32, device=dev)
    ob = torch.empty(B, ncell, dtype=torch.bool, device=dev)
    if B == 0:
        return bev, ob
    nr = len(rows)
    slot = _NODE_SLOTS[_NODE_TURN[0]]
    _NODE_TURN[0] ^= 1
    host, table = slot.acquire(32 * nr + 4 * (B + 1), dev)
    h = host.numpy()
    if nr:
        h[:32 * nr].view(np.int64).reshape(nr, 4)[:] = rows
    h[32 * nr:32 * nr + 4 * (B + 1)].view(np.int32)[:] = offs
    rc = lib.bb_bev_splat_nodes(host.data_ptr(), nr, host.data_ptr() + 32 * nr, B, table.data_ptr(),
                                S_w2c.contiguous().data_ptr(), T_w2c.contiguous().data_ptr(), C, int(fdt == BF16),
                                map_dim, map_res, y_clip, bev.data_ptr(), ob.data_ptr(), _stream())
    slot.mark_busy()
    _lib.check(rc, "bb_bev_splat_nodes")
    return bev, ob


def bev_lift_points(depths, T_c2w, world_shift, depth_scale, fx, fy, cx, cy):
    """World points of N depth views (bb_bev_lift_points): depths f32 (N, Hf, Wf) stored units, T_c2w f32 (N, 4, 4),
    world_shift f32 (3,), all contiguous on one device -> (pts f32 (N, Hf*Wf, 3), no_depth bool (N, Hf*Wf))."""
    for t, n in ((depths, "depths"), (T_c2w, "T_c2w"), (world_shift, "world_shift")):
        _req(t, torch.float32, n)
        if not t.is_contiguous():
            raise ValueError("%s must be contiguous" % n)
        if t.device != depths.device:
            raise ValueError("%s must be on %s, got %s" % (n, depths.device, t.device))
    if depths.dim() != 3 or T_c2w.shape != (depths.shape[0], 4, 4) or world_shift.shape != (3,):
        raise ValueError("want depths (N, Hf, Wf), T_c2w (N, 4, 4) and world_shift (3,), got %s, %s and %s"
                         % (tuple(depths.shape), tuple(T_c2w.shape), tuple(world_shift.shape)))
    N, Hf, Wf = depths.shape
    pts = torch.empty(N, Hf * Wf, 3, dtype=torch.float32, device=depths.device)
    nod = torch.empty(N, Hf * Wf, dtype=torch.bool, device=depths.device)
    _lib.check(_lib.load().bb_bev_lift_points(depths.data_ptr(), T_c2w.data_ptr(), N, Hf, Wf, depth_scale, fx, fy, cx,
                                              cy, world_shift.data_ptr(), pts.data_ptr(), nod.data_ptr(), _stream()),
               "bb_bev_lift_points")
    return pts, nod
