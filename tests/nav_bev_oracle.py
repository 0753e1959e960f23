"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the agents' per-step BEV input (map_nav_src), the oracle of
bb_bev_splat_nodes and bevbert_b200.agent_bev.  Built on the discretisation and scatter-mean of oracle/bevbert_ref.py;
every function cites the reference lines it restates (paths relative to the reference root).  Pinned to the reference's
own GraphMap and project_bev by tests/golden/nav_bev.pt (tests/golden/make_nav_bev_golden.py).  The product never
imports it."""
import torch

from oracle.bevbert_ref import cell_index, scatter_mean

def gather_nodes(gmap, vp, order):
    """GraphMap.gather_node_pc's selection (map_nav_src/models/graph_utils.py:129-143): the node alone at order 0, else
    every node with a cloud whose graph path from vp has at most `order` hops, in node_pc insertion order."""
    if order == 0:
        return [vp]
    return [c for c in gmap.node_pc.keys() if len(gmap.graph.path(vp, c)) <= order]


def heading_T(headings):
    """transfrom3D (map_nav_src/models/bev_utils.py:7-36) for (x, y, z, heading, elevation) = (0, 0, 0, h, 0), as
    agent.py:156-159 builds it: float64 entries, then float32.  (B,) -> (B,4,4)"""
    import numpy as np
    h = np.asarray(headings, dtype=np.float64)
    cx, sx, cy, sy = np.cos(0.0), np.sin(0.0), np.cos(h), np.sin(h)
    T = np.zeros([h.shape[0], 4, 4])
    T[:, 0, 0], T[:, 0, 1], T[:, 0, 2] = cy, sx * sy, cx * sy
    T[:, 1, 1], T[:, 1, 2] = cx, -sx
    T[:, 2, 0], T[:, 2, 1], T[:, 2, 2] = -sy, cy * sx, cy * cx
    T[:, 3, 3] = 1
    return torch.from_numpy(T.astype(np.float32))


def nav_cell_index(nodes, S, E, D, res, y_clip=0.5):
    """One sample of the agents' splat (agent.py:161-166) on the concatenation gather_node_pc builds
    (graph_utils.py:139-141): pc - S, then the 4-term dot products with T_w2c rows in the fixed left-to-right order of
    lift_points (the reference leaves it to matmul), then cell_index.  nodes: (pc (n,3), mask (n,), feat (n,C)).
    -> (cell index (P,) int64 with -1 = dropped, features (P,C) f32)."""
    pc = torch.cat([n[0].float().cpu() for n in nodes], 0)
    nod = torch.cat([n[1].bool().cpu() for n in nodes], 0)
    feat = torch.cat([n[2].float().cpu() for n in nodes], 0)
    S, E = S.float().cpu(), E.float().cpu()
    p = [pc[:, j] - S[j] for j in range(3)]
    e = []
    for j in range(3):
        acc = p[0] * E[j, 0]
        acc = acc + p[1] * E[j, 1]
        acc = acc + p[2] * E[j, 2]
        acc = acc + E[j, 3]
        e.append(acc)
    ego = torch.stack(e, -1)
    idx = cell_index(ego, nod, D, res, y_clip)
    # NaN coordinates pass every comparison in the reference and then index out of range; they are dropped here
    return torch.where(torch.isnan(ego[:, 0]) | torch.isnan(ego[:, 2]), torch.full_like(idx, -1), idx), feat


def nav_splat_nodes(clouds, S_w2c, T_w2c, D, res, y_clip=0.5):
    """gather_node_pc's torch.cat + pad_sequence (agent.py:323-325) + splat + project_bev
    (map_nav_src/models/bev_utils.py:382-417) on CPU.  clouds[b]: list of (pc (n,3), mask (n,), feat (n,C)) node
    tuples in gather order.  Padding points are no-depth points and drop out, so each sample is pooled from its own
    concatenated cloud.  -> (bev (B, D*D, C) f32, ob_mask (B, D*D) bool); a sample without nodes gives zeros."""
    C = next((int(n[2].shape[1]) for nodes in clouds for n in nodes), None)
    bevs, obs = [], []
    for b, nodes in enumerate(clouds):
        if not nodes:
            bevs.append(torch.zeros(D * D, C))
            obs.append(torch.zeros(D * D, dtype=torch.bool))
            continue
        idx, feat = nav_cell_index(nodes, S_w2c.reshape(-1, 3)[b], T_w2c.reshape(-1, 4, 4)[b], D, res, y_clip)
        bev = scatter_mean(feat, idx, D * D)
        bevs.append(bev)
        obs.append(~((bev.max(-1)[0] == 0) & (bev.min(-1)[0] == 0)))
    return torch.stack(bevs, 0), torch.stack(obs, 0)


def nav_bev_variable(obs, gmaps, pc_order, D, res, map_cand_to_bev, bev_pos):
    """LocalAgent._nav_bev_variable (map_nav_src/r2r/agent.py:293-337; reverie/agent_obj.py the same) with the splat of
    nav_splat_nodes: the dict the navigation call takes, on CPU."""
    import numpy as np
    clouds, nav_masks, cand_idxs, cand_vpids, gpos = [], [], [], [], []
    for ob, gmap in zip(obs, gmaps):
        clouds.append([gmap.node_pc[c] for c in gather_nodes(gmap, ob["viewpoint"], pc_order)])
        cand_vpids.append([None] + [c["viewpointId"] for c in ob["candidate"]])
        pos = map_cand_to_bev(ob)
        idx = np.insert(pos[:, 1] * D + pos[:, 0], 0, (D * D - 1) // 2)
        m = np.zeros(D * D, dtype=bool)
        m[idx] = True
        nav_masks.append(torch.from_numpy(m))
        cand_idxs.append(torch.from_numpy(idx))
        gpos.append(torch.from_numpy(gmap.get_pos_fts(ob["viewpoint"], [gmap.start_vp], ob["heading"], ob["elevation"])))
    B = len(obs)
    S = torch.from_numpy(np.vstack([[np.array([o["position"][0], o["position"][2], -o["position"][1]])]
                                    for o in obs]).astype(np.float32))
    T = heading_T([o["heading"] for o in obs])
    bev, _ = nav_splat_nodes(clouds, S, T, D, res)
    L = max(len(c) for c in cand_idxs)
    cidx = torch.zeros(B, L, dtype=cand_idxs[0].dtype)
    for i, c in enumerate(cand_idxs):
        cidx[i, :len(c)] = c
    g = torch.stack(gpos, 0).expand(-1, D * D, -1)
    return {"bev_fts": bev, "bev_pos_fts": torch.cat([g, bev_pos.cpu().reshape(B, -1, 3)], -1),
            "bev_masks": torch.ones(B, D * D, dtype=torch.bool), "bev_nav_masks": torch.stack(nav_masks, 0),
            "bev_cand_idxs": cidx, "bev_cand_vpids": cand_vpids}
