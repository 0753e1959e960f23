"""Synthetic navigation episodes for the agent-side BEV tests (tests/test_nav_bev_*.py,
tests/golden/make_nav_bev_golden.py).

A house is a G x G grid of viewpoints 1.25 m apart (positions exact in float32, so that at heading 0 the ego transform
is exact and hand-placed points land on exact cell edges).  Each sample walks the grid for `steps` steps and leaves one
point cloud per visit, as the agents' `lift` does (map_nav_src/r2r/agent.py:493-501): sample 0 walks a snake that
visits a new viewpoint at every step (more than 21 nodes by step 22), sample 1 a seeded random walk with revisits,
sample 2 goes back and forth between two viewpoints.  Everything is regenerated bit-identically from the seed.
"""
import numpy as np
import torch

from bevbert_b200 import synth

GRID = 6
SPACING = 1.25


def vp_name(r, c):
    return "v%d_%d" % (r, c)


def vp_rc(vp):
    r, c = vp[1:].split("_")
    return int(r), int(c)


def vp_position(vp):
    r, c = vp_rc(vp)
    return [c * SPACING, r * SPACING, 1.5]           # simulator (x, y, z); the agents' world frame is (x, z, -y)


def neighbours(vp):
    r, c = vp_rc(vp)
    return [vp_name(r + dr, c + dc) for dr, dc in ((-1, 0), (0, 1), (1, 0), (0, -1))
            if 0 <= r + dr < GRID and 0 <= c + dc < GRID]


def walk(sample, steps, seed):
    if sample % 3 == 0:      # snake: a new viewpoint at every step
        cells = [(r, c if r % 2 == 0 else GRID - 1 - c) for r in range(GRID) for c in range(GRID)]
        return [vp_name(*cells[t % len(cells)]) for t in range(steps)]
    if sample % 3 == 2:      # back and forth
        return [vp_name(2, 2 + t % 2) for t in range(steps)]
    vps = [vp_name(1, 1)]
    pick = synth.det_randint((steps,), seed, 50 + sample, 0, 3)
    for t in range(1, steps):
        nb = neighbours(vps[-1])
        vps.append(nb[int(pick[t]) % len(nb)])
    return vps


def heading(sample, t, seed):
    if (sample + t) % 4 == 0:
        return 0.0           # exact ego transform: the hand-placed edge points stay on their edges
    return float(synth.det_uniform((1,), seed, 1000 * sample + t, -np.pi, np.pi)[0])


def make_ob(vp, hd):
    return {"viewpoint": vp, "position": vp_position(vp), "heading": hd, "elevation": 0.0,
            "candidate": [{"viewpointId": n, "position": vp_position(n)} for n in neighbours(vp)]}


def node_cloud(vp, sample, t, seed, C=768, n=None, feat_dtype=torch.float32):
    """world-frame cloud (n,3) f32 around vp, no-depth mask (n,) bool, features (n,C): points up to 6.5 m away (some
    outside a 21 x 0.5 m map), heights across the 0.5 m clip, ~5 % without depth, and hand-placed points on exact .5
    cell edges and at y == 0.5 relative to the node."""
    s = seed * 7919 + sample * 131 + t
    if n is None:
        n = 40 + (7 * t + 13 * sample) % 29
    x, y, z = vp_position(vp)
    S = torch.tensor([x, z, -y], dtype=torch.float32)
    off = synth.det_uniform((n, 3), s, 1, -6.5, 6.5)
    off[:, 1] = synth.det_uniform((n,), s, 2, -1.5, 1.0)
    edge = torch.tensor([[0.25, 0.0, 0.75], [-0.25, 0.5, -1.25], [5.25, 0.1, -5.25], [-5.25, 0.2, 5.24],
                         [0.0, 0.5, 0.0], [5.26, 0.0, 0.25]])
    m = min(n, edge.shape[0])
    off[:m] = edge[:m]
    pc = (S + off).contiguous()
    nod = synth.det_uniform((n,), s, 3) < 0.05
    feat = synth.det_uniform((n, C), s, 4, -1.7, 1.7).to(feat_dtype)
    return pc, nod, feat


def episode(B=3, steps=24, seed=11, C=768):
    """[(obs, clouds, order)] per step: obs of the B samples, the cloud each sample left at this step, pc_order."""
    walks = [walk(i, steps, seed) for i in range(B)]
    out = []
    for t in range(steps):
        obs = [make_ob(walks[i][t], heading(i, t, seed)) for i in range(B)]
        clouds = [node_cloud(walks[i][t], i, t, seed, C) for i in range(B)]
        order = 30 if t == steps - 1 else t % 3
        out.append((obs, clouds, order))
    return out


# --------------------------------------------------------------------------------------------- stub agent and map
class HopGraph:
    """graph.path stand-in: shortest hop paths (BFS) over the edges added so far; path(x, x) = []."""

    def __init__(self):
        self.adj = {}

    def add_edge(self, a, b):
        self.adj.setdefault(a, set()).add(b)
        self.adj.setdefault(b, set()).add(a)

    def path(self, x, y):
        if x == y:
            return []
        prev, frontier = {x: None}, [x]
        while frontier and y not in prev:
            nxt = []
            for u in frontier:
                for v in sorted(self.adj.get(u, ())):
                    if v not in prev:
                        prev[v] = u
                        nxt.append(v)
            frontier = nxt
        if y not in prev:
            return [y]
        p = [y]
        while prev[p[-1]] != x:
            p.append(prev[p[-1]])
        return p[::-1]


class StubGraphMap:
    """The parts of map_nav_src/models/graph_utils.GraphMap the BEV input reads: node_pc (insertion-ordered),
    graph.path, start_vp, get_pos_fts."""

    def __init__(self, start_vp, graph=None):
        self.start_vp = start_vp
        self.node_pc = {}
        self.graph = graph if graph is not None else HopGraph()

    def update_graph(self, ob):
        for c in ob["candidate"]:
            self.graph.add_edge(ob["viewpoint"], c["viewpointId"])

    def update_node_pc(self, vp, pc, pc_mask, pc_feat):
        self.node_pc[vp] = [pc, pc_mask, pc_feat]

    def get_pos_fts(self, cur_vp, gmap_vpids, cur_heading, cur_elevation):
        a, b = np.array(vp_position(cur_vp)), np.array(vp_position(gmap_vpids[0]))
        d = b - a
        return np.array([[np.sin(cur_heading), np.cos(cur_heading), 0.0, 1.0, np.linalg.norm(d) / 30,
                          len(self.graph.path(cur_vp, gmap_vpids[0])) / 10, d[0] / 30]], dtype=np.float32)


class StubArgs:
    def __init__(self, pc_order):
        self.pc_order = pc_order


class StubAgent:
    """bev_dim / bev_res / bev_pos / args.pc_order and a candidate-to-cell map, as the reference agents hold them."""

    def __init__(self, B, D=21, res=0.5, pc_order=1, device="cpu"):
        from bevbert_b200.model.bev_utils import bevpos_polar
        self.bev_dim, self.bev_res = D, res
        self.args = StubArgs(pc_order)
        self.bev_pos = bevpos_polar(D).to(device)[None].expand(B, -1, -1, -1)

    def _map_cand_to_bev(self, ob):
        p = np.array([c["position"] for c in ob["candidate"]], dtype=np.float32)
        x, y = np.float32(ob["position"][0]), np.float32(ob["position"][1])
        g = np.round(np.stack([(p[:, 0] - x), -(p[:, 1] - y)], 1) / self.bev_res) + (self.bev_dim - 1) // 2
        return np.clip(g, 0, self.bev_dim - 1).astype(np.int64)


def run_stub_episode(B=3, steps=24, seed=11, C=768, device="cpu", feat_dtype=torch.float32):
    """Yields (obs, gmaps, order) per step with the stub maps updated as the agents do before _nav_bev_variable."""
    ep = episode(B, steps, seed, C)
    gmaps = [StubGraphMap(ep[0][0][i]["viewpoint"]) for i in range(B)]
    for obs, clouds, order in ep:
        for i, (ob, gm) in enumerate(zip(obs, gmaps)):
            gm.update_graph(ob)
            pc, nod, ft = clouds[i]
            gm.update_node_pc(ob["viewpoint"], pc.to(device), nod.to(device), ft.to(feat_dtype).to(device))
        yield obs, gmaps, order
