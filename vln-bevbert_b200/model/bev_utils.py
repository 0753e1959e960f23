"""BEV lifting on the H100 kernels: same entry points as pretrain_src/model/bev_utils.py
(`bevpos_polar`, `PointCloud.forward`, `PointCloud.project_bev`) plus the fused `lift_splat` used by the
pre-training wrapper (pretrain_cmt.py:114-167)."""
import math

import torch

from .. import bev_nodes
from .. import kernels as K


def bevpos_polar(map_dim):
    """(D, D, 3) [cos, sin, dist/(D/2)] polar position code, centre cell = 0 (bev_utils.py:39-58)."""
    lin = torch.linspace(0.5, map_dim - 0.5, map_dim, dtype=torch.float32)
    ry, rx = torch.meshgrid(lin, lin, indexing="ij")
    ry = -(ry - map_dim / 2)
    rx = rx - map_dim / 2
    dis = (ry ** 2 + rx ** 2) ** 0.5
    c, s = rx / dis, ry / dis
    c[dis == 0] = 0
    s[dis == 0] = 0
    return torch.stack([c, s, dis / (map_dim / 2)], dim=-1)


class PointCloud:
    """Un-projects depth pixels and pools their features into the metric map (bev_utils.py:297-430).

    `forward(depth, T)` returns the world-frame points like the reference; `project_bev` takes an ego-frame
    cloud.  The pre-training path uses `lift_splat`, which fuses both transforms and the cell index into one
    kernel and never materialises the point cloud.
    """

    def __init__(self, vfov, batch_size, feature_map_height, feature_map_width, map_dim, map_res,
                 world_shift_origin=None, z_clip_threshold=0.5, device=None):
        self.fmh, self.fmw = feature_map_height, feature_map_width
        self.map_dim, self.map_res = map_dim, map_res
        self.z_clip_threshold = z_clip_threshold
        hfov = feature_map_width / feature_map_height * vfov
        # float32 like torch.Tensor([[f_x, ...]]) in compute_intrinsic_matrix (bev_utils.py:91-100)
        self.fx = float(torch.tensor(feature_map_width / (2.0 * math.tan(hfov / 2.0)), dtype=torch.float32))
        self.fy = float(torch.tensor(feature_map_height / (2.0 * math.tan(vfov / 2.0)), dtype=torch.float32))
        self.cx, self.cy = feature_map_width / 2.0, feature_map_height / 2.0

    def lift_index(self, depths, T_c2w, S_w2c, T_w2c, depth_scale=10.0, want_pc=False):
        """depths (B,V,1,Hf,Wf) stored units -> int32 cell index (B, V*Hf*Wf) (-1 = dropped) [+ ego cloud]."""
        B, V = depths.shape[0], depths.shape[1]
        d = depths.reshape(B, V, self.fmh, self.fmw)
        return K.bev_lift_index(d, T_c2w.reshape(B, V, 4, 4), S_w2c.reshape(B, 3), T_w2c.reshape(B, 4, 4),
                                self.map_dim, self.map_res, depth_scale, self.fx, self.fy, self.cx, self.cy,
                                self.z_clip_threshold, want_pc)

    def forward(self, depth, T):
        """(N,1,Hf,Wf) metres, (N,4,4) -> world points (N,Hf,Wf,3), no-depth mask (bev_utils.py:349-378)."""
        N = depth.shape[0]
        eye = torch.eye(4, dtype=torch.float32, device=depth.device)[None].repeat(N, 1, 1)
        zero = torch.zeros(N, 3, dtype=torch.float32, device=depth.device)
        _, pc = K.bev_lift_index(depth.reshape(N, 1, self.fmh, self.fmw), T.reshape(N, 1, 4, 4), zero, eye,
                                 self.map_dim, self.map_res, 1.0, self.fx, self.fy, self.cx, self.cy,
                                 self.z_clip_threshold, True)
        return pc.reshape(N, self.fmh, self.fmw, 3), depth[:, 0] == 0

    @torch.no_grad()
    def project_bev(self, pc, no_depth_mask, pc_feat, pc_sem=None):
        """Reference entry point, both variants: pre-training `project_bev(pc, mask, feat, sem)` ->
        (bevs (B,D,D,C), ob_masks (B,D,D), sems (B,D,D,S), sem_masks (B,D,D)) (pretrain_src/model/bev_utils.py:381-430)
        and agent-side `project_bev(pc, mask, feat)` -> (bevs, ob_masks) (map_nav_src/models/bev_utils.py:382-417,
        called at map_nav_src/r2r/agent.py:170).  pc (B,N,3) ego-frame points, no_depth_mask (B,N) bool, pc_feat
        (B,N,C) fp32, pc_sem (B,N,S) fp64 one-hots.  Ragged inputs (a python list of per-sample tensors, as the agents
        build them from neighbouring panoramas) are pooled where they lie, one node per sample with the identity ego
        transform (`splat_nodes`): the same result as padding them with no-depth points.  With semantics they are
        padded that way."""
        if isinstance(pc, (list, tuple)):
            if pc_sem is not None:
                pad = torch.nn.utils.rnn.pad_sequence
                return self.project_bev(pad(list(pc), batch_first=True),
                                        pad([m.bool() for m in no_depth_mask], batch_first=True, padding_value=True),
                                        pad(list(pc_feat), batch_first=True), pad(list(pc_sem), batch_first=True))
            B = len(pc)
            dev = pc[0].device
            S = torch.zeros(B, 3, dtype=torch.float32, device=dev)
            T = torch.eye(4, dtype=torch.float32, device=dev).expand(B, 4, 4)
            clouds = [[(p.float().contiguous(), m.bool().contiguous(),
                        (f if f.dtype == torch.bfloat16 else f.float()).contiguous())]
                      for p, m, f in zip(pc, no_depth_mask, pc_feat)]
            bev, ob = self.splat_nodes(clouds, S, T)
            D = self.map_dim
            return bev.view(B, D, D, -1), ob
        D = self.map_dim
        B = pc.shape[0]
        idx = K.bev_cell_index(pc.float(), no_depth_mask, D, self.map_res, self.z_clip_threshold)
        bev, _, ob, sem, sem_mask = self.splat(idx, pc_feat.float() if pc_feat.dtype != torch.bfloat16 else pc_feat, pc_sem)
        bevs, ob_masks = bev.view(B, D, D, -1), ob.view(B, D, D)
        if pc_sem is None:
            return bevs, ob_masks
        return bevs, ob_masks, sem.view(B, D, D, -1), sem_mask.view(B, D, D)

    @torch.no_grad()
    def splat_nodes(self, clouds, S_w2c, T_w2c):
        """Agent-side BEV straight from the navigation graph's node clouds: `clouds[b]` is the list of
        `(pc, pc_mask, pc_feat)` tuples that `GraphMap.node_pc` holds for the nodes sample b gathers, in gather order
        (world-frame points (n,3), no-depth mask (n,), features (n,C) fp32 or bf16, as `forward` and the agents' `lift`
        produce them); S_w2c (B,3), T_w2c (B,4,4) the agents' ego transform.  One kernel replaces
        `GraphMap.gather_node_pc` + `pad_sequence` + `splat` + `project_bev` (map_nav_src/r2r/agent.py:143-192,293-330)
        with the same result bit for bit, given the fixed-order ego transform.
        -> (bev_fts (B, D*D, C) fp32, ob_masks (B, D, D) bool)."""
        D = self.map_dim
        bev, ob = bev_nodes.bev_splat_nodes(clouds, S_w2c.reshape(-1, 3), T_w2c.reshape(-1, 4, 4), D, self.map_res,
                                            self.z_clip_threshold)
        return bev, ob.view(-1, D, D)

    @torch.no_grad()
    def splat(self, cell_idx, pc_feat, pc_sem=None, want_bf16=False):
        """Pools (B,P,C) fp32 features (and (B,P,S) fp64 labels) into the D*D cells given the cell index."""
        ncell = self.map_dim * self.map_dim
        bev, bev16, ob, _ = K.bev_scatter_mean(pc_feat, cell_idx, ncell, True, want_bf16)
        sem = sem_mask = None
        if pc_sem is not None:
            sem, sem_mask = K.bev_scatter_sem(pc_sem, cell_idx, ncell)
        return bev, bev16, ob, sem, sem_mask
