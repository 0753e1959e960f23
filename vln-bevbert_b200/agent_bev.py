"""The agents' per-step BEV input built by one kernel straight from the navigation graph's node clouds.

`nav_bev_variable(agent, obs, gmaps)` returns the dict of the reference agents' `_nav_bev_variable`
(map_nav_src/r2r/agent.py:293-337, identical in reverie/agent_obj.py, which the SOON agent inherits):
`bev_fts, bev_pos_fts, bev_masks, bev_nav_masks, bev_cand_idxs, bev_cand_vpids`.  Only the point-cloud half changes:
instead of `torch.cat`-ing the clouds of the current node and its neighbours (`GraphMap.gather_node_pc`), padding them
into a batch (`pad_sequence`), transforming them to the ego frame (`splat`) and pooling them (`project_bev`), one
`bb_bev_splat_nodes` launch reads every node cloud where `GraphMap.node_pc` keeps it.  Everything else goes through the
agent's own methods (`_map_cand_to_bev`, `GraphMap.get_pos_fts`, `graph.path`, `bev_pos`, `args.pc_order`).

Install on an agent once it is built:

    agent._nav_bev_variable = types.MethodType(nav_bev_variable, agent)

`ce_nav_bev_variable(trainer, cur_vp, cur_pos, cur_ori)` does the same for the VLN-CE trainer's `_nav_bev_variable`
(bevbert_ce/vlnce_baselines/ss_trainer_BEV.py:477-532); see its docstring.
"""
import importlib
import math
import sys

import numpy as np
import torch

from . import bev_nodes

Y_CLIP = 0.5    # height clip of the agents' project_bev (map_nav_src/models/bev_utils.py:398)


def gathered_nodes(gmap, vp, order, path=None):
    """The viewpoints whose clouds `GraphMap.gather_node_pc(vp, order)` concatenates, in its order: the node alone at
    order 0, otherwise every node with a cloud, in insertion order of `node_pc`, at most `order` graph hops from vp.
    `path(vp, c)`: the shortest path the graph map keeps (default `gmap.graph.path`, the discrete agents')."""
    if order == 0:
        return [vp]
    path = path or gmap.graph.path
    return [c for c in gmap.node_pc if len(path(vp, c)) <= order]


def ego_frames(obs):
    """World -> ego transform of each sample, float32: S (B,3) = (x, z, -y) of the agent's position and T (B,4,4) a
    rotation about the vertical axis by the heading, built in float64 and rounded to float32 like the agents'
    matrices (agent.py:150-159)."""
    S = np.array([[o["position"][0], o["position"][2], -o["position"][1]] for o in obs], dtype=np.float64)
    return heading_frames(S, np.array([o["heading"] for o in obs], dtype=np.float64))


def frames64(xyzhe):
    """transfrom3D (bev_utils.py:7-37 of both trees) before its rounding to float32: (N,5) float64 x, y, z, heading,
    elevation -> (N,4,4) float64 matrices, every entry the same float64 expression as there."""
    cx, sx = np.cos(xyzhe[:, 4]), np.sin(xyzhe[:, 4])
    cy, sy = np.cos(xyzhe[:, 3]), np.sin(xyzhe[:, 3])
    T = np.zeros((len(xyzhe), 4, 4), dtype=np.float64)
    T[:, 0, 0], T[:, 0, 1], T[:, 0, 2], T[:, 0, 3] = cy, sx * sy, cx * sy, xyzhe[:, 0]
    T[:, 1, 1], T[:, 1, 2], T[:, 1, 3] = cx, -sx, xyzhe[:, 1]
    T[:, 2, 0], T[:, 2, 1], T[:, 2, 2], T[:, 2, 3] = -sy, cy * sx, cy * cx, xyzhe[:, 2]
    T[:, 3, 3] = 1.0
    return T


def heading_frames(S, h):
    """(S, T) float32 from float64 positions S (B,3) and headings h (B,): T rotates about the vertical axis by h
    (transfrom3D at zero elevation and translation)."""
    xyzhe = np.zeros((len(h), 5), dtype=np.float64)
    xyzhe[:, 3] = h
    return S.astype(np.float32), frames64(xyzhe).astype(np.float32)


def nav_bev_variable(agent, obs, gmaps):
    """Drop-in for the agents' `_nav_bev_variable(obs, gmaps)`; see the module docstring."""
    B, D = len(obs), agent.bev_dim
    clouds = [[gmap.node_pc[c] for c in gathered_nodes(gmap, ob["viewpoint"], agent.args.pc_order)]
              for ob, gmap in zip(obs, gmaps)]
    dev = next((n[0].device for nodes in clouds for n in nodes), agent.bev_pos.device)

    nav_masks = np.zeros((B, D * D), dtype=bool)
    cand_idxs, cand_vpids, gpos = [], [], []
    for i, (ob, gmap) in enumerate(zip(obs, gmaps)):
        cand_vpids.append([None] + [c["viewpointId"] for c in ob["candidate"]])     # None: the stop action
        pos = agent._map_cand_to_bev(ob)
        idx = np.insert(pos[:, 1] * D + pos[:, 0], 0, (D * D - 1) // 2)            # stop sits on the centre cell
        nav_masks[i, idx] = True
        cand_idxs.append(idx)
        gpos.append(gmap.get_pos_fts(ob["viewpoint"], [gmap.start_vp], ob["heading"], ob["elevation"]))

    S, T = ego_frames(obs)
    frames = torch.from_numpy(np.concatenate([S.ravel(), T.ravel()])).to(dev)     # one upload for both
    bev_fts, _ = bev_nodes.bev_splat_nodes(clouds, frames[:3 * B].view(B, 3), frames[3 * B:].view(B, 4, 4), D,
                                           agent.bev_res, Y_CLIP)

    L = max(len(c) for c in cand_idxs)
    bev_cand_idxs = torch.zeros(B, L, dtype=torch.from_numpy(cand_idxs[0]).dtype)
    for i, c in enumerate(cand_idxs):
        bev_cand_idxs[i, :len(c)] = torch.from_numpy(c)
    gpos = torch.from_numpy(np.stack(gpos, 0)).to(dev)
    return {
        "bev_fts": bev_fts,
        "bev_pos_fts": torch.cat([gpos.expand(-1, D * D, -1), agent.bev_pos.reshape(B, -1, 3)], -1),
        "bev_masks": torch.ones(B, D * D, dtype=torch.bool, device=dev),
        "bev_nav_masks": torch.from_numpy(nav_masks).to(dev),
        "bev_cand_idxs": bev_cand_idxs,
        "bev_cand_vpids": cand_vpids,
    }


def _trainer_heading_fn(trainer):
    """The `heading_from_quaternion` the trainer's own code uses: the one imported by the module of its class or of the
    nearest base class (ss_trainer_BEV.py:61), else graph_utils' (where ss_trainer_BEV takes it from)."""
    for cls in type(trainer).__mro__:
        fn = getattr(sys.modules.get(cls.__module__), "heading_from_quaternion", None)
        if fn is not None:
            return fn
    return importlib.import_module("vlnce_baselines.models.graph_utils").heading_from_quaternion


LIFT_VIEWS, LIFT_GRID, LIFT_DIM = 12, 14, 768       # lift's views, depth-grid side and feature width (:389,402,407)


def lift_frames(cur_pos, headings):
    """`lift`'s camera-to-world fan (ss_trainer_BEV.py:391-399): per environment the 12 views at headings
    -arange(12) * radians(30) + heading, elevation pi and translation (x, y, z), built in float64 as there and rounded
    to float32 like transfrom3D -> (B * 12, 4, 4) float32.  `headings[i]`: heading_from_quaternion(cur_ori[i])."""
    xyzhe = np.zeros([len(cur_pos), LIFT_VIEWS, 5])
    for i, (pos_i, h) in enumerate(zip(cur_pos, headings)):
        x, y, z = pos_i
        xyzhe[i, :, 0] = x
        xyzhe[i, :, 1] = y
        xyzhe[i, :, 2] = z
        xyzhe[i, :, 3] = -np.arange(LIFT_VIEWS) * np.radians(30) + h
        xyzhe[i, :, 4] = np.pi
    return frames64(xyzhe.reshape(-1, 5)).astype(np.float32)


def lift_intrinsics(projector):
    """(fx, fy, cx, cy) of the trainer's PointCloud as its `forward` uses them: compute_intrinsic_matrix
    (bev_utils.py:91-100) in float64, rounded to float32 by torch.Tensor.  Raises ValueError for a projector whose
    `forward` bb_bev_lift_points does not reproduce: a feature map other than lift's 14 x 14, or a world_shift_origin
    other than three float32 values."""
    fmh, fmw, vfov = projector.fmh, projector.fmw, projector.vfov
    if (fmh, fmw) != (LIFT_GRID, LIFT_GRID):
        raise ValueError("lift reads 14 x 14 depth grids; the projector's feature map is %s x %s" % (fmh, fmw))
    if not isinstance(vfov, (int, float)) or not 0.0 < vfov < math.pi:
        raise ValueError("projector.vfov must be a field of view in (0, pi) radians, got %r" % (vfov,))
    shift = projector.world_shift_origin
    if not (torch.is_tensor(shift) and shift.dtype == torch.float32 and shift.numel() == 3 and shift.shape[-1] == 3):
        raise ValueError("projector.world_shift_origin must be a float32 tensor of three values, got %r" % (shift,))
    hfov = fmw / fmh * vfov
    K = [fmw / (2.0 * math.tan(hfov / 2.0)), fmh / (2.0 * math.tan(vfov / 2.0)), fmw / 2.0, fmh / 2.0]
    return tuple(torch.tensor(K, dtype=torch.float32).tolist())


def ce_lift(trainer, cur_pos, cur_ori, rgb_grid, depth_grid):
    """Drop-in for the VLN-CE trainer's `lift(cur_pos, cur_ori, rgb_grid, depth_grid)` (ss_trainer_BEV.py:386-410),
    same (pc (B, 2352, 3), pc_mask (B, 2352), pc_feat (B, 2352, 768)).  The heading fan is `lift_frames` with the
    trainer's own `heading_from_quaternion` (`_trainer_heading_fn`), uploaded in one copy; one `bb_bev_lift_points`
    launch then does `PointCloud.forward` (bev_utils.py:349-378) on `depth_grid * 10` with the trainer's projector
    (`lift_intrinsics`), the camera-to-world product in the kernel's fixed fp32 order where the reference calls bmm.
    pc_feat is a view of rgb_grid, as in the reference.  depth_grid: contiguous float32 CUDA tensor of B * 12 * 196
    values (the waypoint step's pano_depth_grid), read in place; rgb_grid on the same device.  Nothing in it
    synchronises with the host.

    Install on the trainer once it is built: graphs.install_ce_lift(trainer)."""
    fx, fy, cx, cy = lift_intrinsics(trainer.projector)
    B = len(cur_pos)
    n = B * LIFT_VIEWS * LIFT_GRID * LIFT_GRID
    if not (torch.is_tensor(depth_grid) and depth_grid.is_cuda and depth_grid.dtype == torch.float32
            and depth_grid.is_contiguous() and depth_grid.numel() == n):
        raise ValueError("depth_grid must be a contiguous float32 CUDA tensor of %d x 12 x 196 values, got %s"
                         % (B, depth_grid.dtype if torch.is_tensor(depth_grid) else type(depth_grid)))
    dev = depth_grid.device
    if rgb_grid.device != dev or trainer.projector.world_shift_origin.device != dev:
        raise ValueError("rgb_grid and projector.world_shift_origin must be on %s" % dev)
    heading_from_quaternion = _trainer_heading_fn(trainer)
    T = torch.from_numpy(lift_frames(cur_pos, [heading_from_quaternion(o) for o in cur_ori]))
    T = T.pin_memory().to(dev, non_blocking=True)
    shift = trainer.projector.world_shift_origin.reshape(3).contiguous()
    pc, pc_mask = bev_nodes.bev_lift_points(depth_grid.view(-1, LIFT_GRID, LIFT_GRID), T, shift, 10.0, fx, fy, cx, cy)
    pc_feat = rgb_grid.reshape(-1, LIFT_GRID, LIFT_GRID, LIFT_DIM).reshape(B, -1, LIFT_DIM)
    return pc.view(B, -1, 3), pc_mask.view(B, -1), pc_feat


def ce_nav_bev_variable(trainer, cur_vp, cur_pos, cur_ori):
    """Drop-in for the VLN-CE trainer's `_nav_bev_variable(cur_vp, cur_pos, cur_ori)` (ss_trainer_BEV.py:477-532),
    same dict.  The clouds of `GraphMap.gather_node_pc(vp, order=1)` (graph_utils.py:332-346: the nodes with a cloud
    whose shortest path from vp has at most one node, i.e. vp itself) are transformed to each sample's ego frame and
    pooled into the `trainer.bev_dim`-square map at `trainer.bev_res` by one `bb_bev_splat_nodes` launch, instead of
    `pad_sequence` + `splat` (:413-463) + `PointCloud.project_bev`.  The ego frame is `splat`'s: S = (x, y, z) of the
    position and T `transfrom3D` of heading -heading_from_quaternion(orientation), with the trainer's own
    `heading_from_quaternion` (`_trainer_heading_fn`); like transfrom3D, T is built in float64 and rounded to float32.
    The node clouds must be float32 points (the kernel transforms them in fp32, in a fixed order).  Candidates
    (`GraphMap.get_neighbors`, the trainer's `_discretize_polar_relpos`) and the global position feature
    (`GraphMap.get_pos_fts` towards the start node '0') come from the trainer's own objects.  `bev_masks` is all True,
    as `splat` returns it without VIDEO_OPTION; `bev_cand_idxs` stays on the host, as the trainer's does (:511).

    Install on the trainer once it is built:

        trainer._nav_bev_variable = types.MethodType(ce_nav_bev_variable, trainer)
    """
    heading_from_quaternion = _trainer_heading_fn(trainer)
    gmaps, D = trainer.gmaps, trainer.bev_dim
    B = len(gmaps)
    clouds = [[tuple(gm.node_pc[c]) for c in gathered_nodes(gm, vp, 1, lambda a, b, gm=gm: gm.shortest_path[a][b])]
              for gm, vp in zip(gmaps, cur_vp)]
    dev = trainer.bev_pos.device

    nav_masks = np.zeros((B, D * D), dtype=bool)
    cand_idxs, cand_vpids, gpos = [], [], []
    for i, gm in enumerate(gmaps):
        vps, relpos = gm.get_neighbors(cur_vp[i], cur_pos[i], cur_ori[i])
        xy = trainer._discretize_polar_relpos(relpos)
        idx = xy[:, 1] * D + xy[:, 0]
        nav_masks[i, idx] = True
        cand_idxs.append(idx)
        cand_vpids.append(vps)
        gpos.append(gm.get_pos_fts(cur_vp[i], cur_pos[i], cur_ori[i], ["0"]))       # '0' is the start node

    S = np.array([[p[0], p[1], p[2]] for p in cur_pos], dtype=np.float64)
    S, T = heading_frames(S, np.array([-heading_from_quaternion(o) for o in cur_ori], dtype=np.float64))
    frames = torch.from_numpy(np.concatenate([S.ravel(), T.ravel()])).to(dev)     # one upload for both
    bev_fts, _ = bev_nodes.bev_splat_nodes(clouds, frames[:3 * B].view(B, 3), frames[3 * B:].view(B, 4, 4), D,
                                           trainer.bev_res, Y_CLIP, C=768)

    L = max(len(c) for c in cand_idxs)
    bev_cand_idxs = torch.zeros(B, L, dtype=torch.from_numpy(cand_idxs[0]).dtype)
    for i, c in enumerate(cand_idxs):
        bev_cand_idxs[i, :len(c)] = torch.from_numpy(c)
    gpos = torch.from_numpy(np.stack(gpos, 0)).to(dev)
    return {
        "bev_fts": bev_fts,
        "bev_pos_fts": torch.cat([gpos.expand(-1, D * D, -1), trainer.bev_pos.expand(B, -1, -1, -1).reshape(B, -1, 3)],
                                 -1),
        "bev_masks": torch.ones(B, D * D, dtype=torch.bool, device=dev),
        "bev_nav_masks": torch.from_numpy(nav_masks).to(dev),
        "bev_cand_idxs": bev_cand_idxs,
        "bev_cand_vpids": cand_vpids,
    }
