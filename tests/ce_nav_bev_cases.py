"""Synthetic VLN-CE episodes for the trainer-side BEV adapter (agent_bev.ce_nav_bev_variable): a stand-in trainer with
the attributes and methods the adapter reads from the CE trainer (ss_trainer_BEV.py:205-218, 465-475) and graph maps
with the GraphMap surface it uses (node_pc, shortest_path, get_neighbors, get_pos_fts; graph_utils.py:155-365).

The agent walks a small grid of waypoints; every step stores the current node's cloud (a revisit overwrites it, as
update_node_pc does), so clouds hold points inside the 11 m map, outside it, above the height clip and without depth.
Orientations are stand-ins: `heading_from_quaternion` below (the adapter takes the trainer module's own) reads the
heading straight from them."""
import math

import networkx as nx
import numpy as np
import torch

from bevbert_b200 import synth
from oracle.bevbert_ref import bevpos_polar

D, RES = 11, 1


def heading_from_quaternion(quat):
    """stand-in for graph_utils.heading_from_quaternion: the orientations here carry the heading in radians"""
    return float(quat[0]) % (2 * np.pi)


def cloud(seed, stream, n, C=768, feat_dtype=torch.float32, device="cpu"):
    """(pc (n,3) world frame around the origin, no-depth (n,), feat (n,C)); y spans the 0.5 m clip"""
    pc = synth.det_uniform((n, 3), seed, stream, -9.0, 9.0)
    pc[:, 1] = synth.det_uniform((n,), seed, stream + 1, -1.5, 1.0)
    nod = synth.det_uniform((n,), seed, stream + 2) < 0.15
    ft = synth.det_uniform((n, C), seed, stream + 3, -2.0, 2.0).to(feat_dtype)
    return pc.to(device), nod.to(device), ft.to(device)


class StubGraphMap:
    def __init__(self):
        self.node_pc, self.node_pos = {}, {}
        self.g = nx.Graph()
        self.shortest_path = {}

    def visit(self, vp, pos, nbrs, pc):
        self.node_pos[vp] = pos
        self.g.add_node(vp)
        for u, upos in nbrs:
            self.node_pos.setdefault(u, upos)
            self.g.add_edge(vp, u, weight=float(np.linalg.norm(np.subtract(pos, upos))))
        self.shortest_path = dict(nx.all_pairs_dijkstra_path(self.g))
        self.node_pc[vp] = list(pc)                 # update_node_pc (graph_utils.py:329-330)

    def get_neighbors(self, cur_vp, cur_pos, cur_ori):
        vps, rel = [None], [np.zeros(2)]
        for vp, p in self.node_pos.items():
            if len(self.shortest_path[cur_vp].get(vp, ())) == 2:
                dx, dz = p[0] - cur_pos[0], p[2] - cur_pos[2]
                rel.append(np.array([math.atan2(dx, -dz) - heading_from_quaternion(cur_ori), math.hypot(dx, dz)],
                                    dtype=np.float32))
                vps.append(vp)
        return vps, np.stack(rel, 0)

    def get_pos_fts(self, cur_vp, cur_pos, cur_ori, gmap_vp_ids):
        h = heading_from_quaternion(cur_ori)
        return np.array([[math.sin(h), math.cos(h), 0.0, 1.0, cur_pos[0] / 10, cur_pos[2] / 10,
                          len(self.node_pc) / 10]], dtype=np.float32)


class StubTrainer:
    def __init__(self, B, device="cpu"):
        self.bev_dim, self.bev_res = D, RES
        self.bev_pos = bevpos_polar(D)[None].to(device)          # 1 x 11 x 11 x 3 (ss_trainer_BEV.py:217-218)
        self.gmaps = [StubGraphMap() for _ in range(B)]

    def _discretize_polar_relpos(self, cands_relpos):          # ss_trainer_BEV.py:465-475
        cx = cy = int((self.bev_dim - 1) // 2)
        x = cx + (cands_relpos[:, 1] * np.sin(cands_relpos[:, 0]) / self.bev_res).round()
        y = cy - (cands_relpos[:, 1] * np.cos(cands_relpos[:, 0]) / self.bev_res).round()
        xy = np.concatenate([x[:, None], y[:, None]], axis=1)
        xy[xy < 0] = 0
        xy[xy >= self.bev_dim] = self.bev_dim - 1
        return xy.astype(np.int64)


def _pos(r, c):
    return np.array([1.7 * c, 0.2 * ((r + c) % 3), -1.3 * r])


def episode(B=3, steps=6, seed=13, device="cpu", feat_dtype=torch.float32, n=700):
    """-> (trainer, per-step (cur_vp, cur_pos, cur_ori)); the trainer's maps evolve as each step is yielded"""
    tr = StubTrainer(B, device)
    walk = [(0, 0), (0, 1), (1, 1), (0, 1), (1, 2), (1, 1)]       # a revisit at steps 3 and 5
    for t in range(steps):
        cur_vp, cur_pos, cur_ori = [], [], []
        for i, gm in enumerate(tr.gmaps):
            r, c = walk[(t + i) % len(walk)]
            vp = "n%d_%d" % (r, c)
            pos = _pos(r, c) + 0.1 * i
            nbrs = [("n%d_%d" % (r + dr, c + dc), _pos(r + dr, c + dc) + 0.1 * i)
                    for dr, dc in ((0, 1), (1, 0), (0, -1), (-1, 0))]
            pc = cloud(seed, 1000 * t + 10 * i, n - 37 * i, feat_dtype=feat_dtype, device=device)
            pc = (pc[0] + torch.tensor(pos, dtype=torch.float32, device=device), pc[1], pc[2])
            gm.visit(vp, pos, nbrs, pc)
            cur_vp.append(vp)
            cur_pos.append(tuple(pos))
            cur_ori.append(np.array([0.4 * t - 1.1 * i, 0.0, 0.0, 1.0]))
        yield tr, cur_vp, cur_pos, cur_ori
