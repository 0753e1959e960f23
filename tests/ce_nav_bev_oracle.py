"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the VLN-CE trainer's per-step BEV input, the oracle of
bevbert_b200.agent_bev.ce_nav_bev_variable.  Paths are relative to bevbert_ce/vlnce_baselines of the reference.

The trainer's `splat` (ss_trainer_BEV.py:413-463) cannot be executed from the reference source: its module imports
habitat_baselines, lmdb, gym and the simulator environments.  It is restated here, with the point transform in the
fixed left-to-right fp32 order of tests/nav_bev_oracle.py (the reference leaves it to matmul).  The pieces it is built
from are pinned to the reference by tests/golden/small_ce_nav.pt: GraphMap.gather_node_pc (graph_utils.py:332-346),
transfrom3D (bev_utils.py:7-37) and PointCloud.project_bev at 11 x 11 / 1 m (bev_utils.py:382-417)."""
import numpy as np
import torch

from nav_bev_oracle import nav_splat_nodes


def gather_nodes(gmap, vp, order):
    """GraphMap.gather_node_pc's selection (graph_utils.py:332-346): the node alone at order 0, else every node with a
    cloud whose shortest path from vp has at most `order` nodes, in node_pc insertion order."""
    if order == 0:
        return [vp]
    return [c for c in gmap.node_pc.keys() if len(gmap.shortest_path[vp][c]) <= order]


def transfrom3D(xyzhe):
    """bev_utils.py:7-37: (N,5) x, y, z, heading, elevation -> (N,4,4), entries in float64 rounded to float32"""
    cx, sx = np.cos(xyzhe[:, 4]), np.sin(xyzhe[:, 4])
    cy, sy = np.cos(xyzhe[:, 3]), np.sin(xyzhe[:, 3])
    T = np.zeros([xyzhe.shape[0], 4, 4])
    T[:, 0, 0], T[:, 0, 1], T[:, 0, 2], T[:, 0, 3] = cy, sx * sy, cx * sy, xyzhe[:, 0]
    T[:, 1, 0], T[:, 1, 1], T[:, 1, 2], T[:, 1, 3] = 0, cx, -sx, xyzhe[:, 1]
    T[:, 2, 0], T[:, 2, 1], T[:, 2, 2], T[:, 2, 3] = -sy, cy * sx, cy * cx, xyzhe[:, 2]
    T[:, 3, 3] = 1
    return T.astype(np.float32)


def splat_frames(cur_pos, headings):
    """splat's S and T (ss_trainer_BEV.py:419-430): S = (x, y, z) as float32, T = transfrom3D of heading -h at zero
    elevation and translation.  `headings`: the heading_from_quaternion of each orientation."""
    S = torch.from_numpy(np.vstack([np.array(p, dtype=np.float64)[None] for p in cur_pos]).astype(np.float32))
    xyzhe = np.zeros([len(headings), 5])
    xyzhe[:, 3] = -np.asarray(headings, dtype=np.float64)
    return S, torch.from_numpy(transfrom3D(xyzhe))


def splat(clouds, S, T, D, res, y_clip=0.5):
    """pad_sequence (no-depth padding) + splat's ego transform + project_bev (:494-496, :432-441): -> (bev (B, D*D, C),
    ob (B, D*D))"""
    return nav_splat_nodes(clouds, S, T, D, res, y_clip)


def ce_nav_bev_variable(gmaps, cur_vp, cur_pos, cur_ori, headings, D, res, discretize, bev_pos):
    """_nav_bev_variable (ss_trainer_BEV.py:477-532) with the splat above; `headings[i]` is heading_from_quaternion of
    cur_ori[i], `discretize` the trainer's _discretize_polar_relpos (:465-475)."""
    clouds, nav_masks, cand_idxs, cand_vpids, gpos = [], [], [], [], []
    for i, gm in enumerate(gmaps):
        clouds.append([tuple(gm.node_pc[c]) for c in gather_nodes(gm, cur_vp[i], 1)])
        vps, relpos = gm.get_neighbors(cur_vp[i], cur_pos[i], cur_ori[i])
        xy = discretize(relpos)
        idx = xy[:, 1] * D + xy[:, 0]
        m = np.zeros(D * D, dtype=bool)
        m[idx] = True
        nav_masks.append(torch.from_numpy(m))
        cand_idxs.append(torch.from_numpy(idx))
        cand_vpids.append(vps)
        gpos.append(torch.from_numpy(gm.get_pos_fts(cur_vp[i], cur_pos[i], cur_ori[i], ["0"])))
    B = len(gmaps)
    S, T = splat_frames(cur_pos, headings)
    bev, _ = splat(clouds, S, T, D, res)
    L = max(len(c) for c in cand_idxs)
    cidx = torch.zeros(B, L, dtype=cand_idxs[0].dtype)
    for i, c in enumerate(cand_idxs):
        cidx[i, :len(c)] = c
    g = torch.stack(gpos, 0).expand(-1, D * D, -1)
    return {"bev_fts": bev, "bev_pos_fts": torch.cat([g, bev_pos.cpu().expand(B, -1, -1, -1).reshape(B, -1, 3)], -1),
            "bev_masks": torch.ones(B, D * D, dtype=torch.bool), "bev_nav_masks": torch.stack(nav_masks, 0),
            "bev_cand_idxs": cidx, "bev_cand_vpids": cand_vpids}
