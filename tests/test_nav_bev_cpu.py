"""Agent-side BEV from node clouds without a GPU: the oracle against the reference's own GraphMap + project_bev
(tests/golden/nav_bev.pt), the agent adapter's host logic (node order, sample offsets, ego frames, the rest of the
dict) against the oracle's restatement of _nav_bev_variable, and the C entry point's host-side argument checks."""
import ctypes
import os

import numpy as np
import pytest
import torch

import nav_bev_cases as NB
import nav_bev_oracle as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nav_bev.pt")


def _splat_nodes_cpu(clouds, S_w2c, T_w2c, map_dim, map_res, y_clip=0.5, C=None):
    """bev_nodes.bev_splat_nodes restated on CPU by the oracle (bb_bev_splat_nodes' contract)"""
    if not any(clouds):
        return torch.zeros(len(clouds), map_dim * map_dim, C), torch.zeros(len(clouds), map_dim * map_dim, dtype=torch.bool)
    return R.nav_splat_nodes(clouds, S_w2c, T_w2c, map_dim, map_res, y_clip)


@pytest.fixture
def splat_cpu(emu, monkeypatch):
    """the kernel emulation of `emu` plus the node splat on CPU; yields the list of (clouds, S, T) it was called with"""
    from bevbert_b200 import bev_nodes
    calls = []

    def spy(clouds, S, T, *a, **k):
        calls.append((clouds, S, T))
        return _splat_nodes_cpu(clouds, S, T, *a, **k)
    monkeypatch.setattr(bev_nodes, "bev_splat_nodes", spy)
    return calls


class _PinnedPaths:
    """graph.path with the path lengths the reference's FloydGraph gave at this step"""

    def __init__(self, vp, keys, hops):
        self.len = {(vp, k): h for k, h in zip(keys, hops)}

    def path(self, x, y):
        return [y] * self.len[(x, y)]


def test_oracle_matches_reference_golden():
    from bevbert_b200.agent_bev import gathered_nodes
    g = torch.load(GOLD, weights_only=False)
    D, res, B = g["D"], g["res"], g["B"]
    ep = NB.episode(B=B)
    assert len(ep) == len(g["steps"])
    gmaps = [NB.StubGraphMap(ep[0][0][i]["viewpoint"]) for i in range(B)]
    flips = total = exact_steps = 0
    for (obs, clouds, order), pin in zip(ep, g["steps"]):
        assert order == pin["order"]
        for i, (ob, gm) in enumerate(zip(obs, gmaps)):
            gm.update_node_pc(ob["viewpoint"], *clouds[i])
            assert list(gm.node_pc.keys()) == pin["keys"][i]
            gm.graph = _PinnedPaths(ob["viewpoint"], pin["keys"][i], pin["hops"][i])
            # the product's selection and the oracle's reproduce the reference's gather_node_pc order and membership
            assert gathered_nodes(gm, ob["viewpoint"], order) == pin["vps"][i]
            assert R.gather_nodes(gm, ob["viewpoint"], order) == pin["vps"][i]
        sel = [[gm.node_pc[v] for v in pin["vps"][i]] for i, gm in enumerate(gmaps)]
        S = torch.tensor([[o["position"][0], o["position"][2], -o["position"][1]] for o in obs], dtype=torch.float32)
        T = R.heading_T([o["heading"] for o in obs])
        bev, ob_mask = R.nav_splat_nodes(sel, S, T, D, res)
        same = True
        for i in range(B):
            idx, _ = R.nav_cell_index(sel[i], S[i], T[i], D, res)
            ref = pin["cell_idx"][i].long()
            flips += int((idx != ref).sum())
            total += idx.numel()
            same &= torch.equal(idx, ref)
        if same:       # the reference's matmul and the fixed order put every point in the same cell
            exact_steps += 1
            assert torch.equal(bev.double().sum(-1), pin["cell_sums"])
            assert torch.equal(bev.reshape(-1, bev.shape[-1])[pin["bev"]["idx"]], pin["bev"]["rows"])
            assert torch.equal(ob_mask, pin["ob_masks"])
    assert flips <= total * 1e-5, "cell-index disagreement with the reference: %d of %d" % (flips, total)
    assert exact_steps >= len(ep) - 2
    assert max(len(v) for v in g["steps"][-1]["vps"]) > 21


def test_adapter_host_logic_equals_oracle(splat_cpu):
    """nav_bev_variable on stub agents and maps, with the kernel replaced by the oracle: the node lists handed to the
    kernel are the map's own tuples in gather order, and the whole dict equals the oracle's _nav_bev_variable."""
    from bevbert_b200.agent_bev import nav_bev_variable
    seen = splat_cpu
    B = 3
    for obs, gmaps, order in NB.run_stub_episode(B=B, steps=24, C=16):
        agent = NB.StubAgent(B, pc_order=order)
        got = nav_bev_variable(agent, obs, gmaps)
        want = R.nav_bev_variable(obs, gmaps, order, agent.bev_dim, agent.bev_res, agent._map_cand_to_bev, agent.bev_pos)
        clouds, S, T = seen[-1]
        for i, (ob, gm) in enumerate(zip(obs, gmaps)):
            vps = R.gather_nodes(gm, ob["viewpoint"], order)
            assert len(clouds[i]) == len(vps) and all(c is gm.node_pc[v] for c, v in zip(clouds[i], vps))
        assert torch.equal(S, torch.tensor([[o["position"][0], o["position"][2], -o["position"][1]] for o in obs]))
        # same cells as the agents' transfrom3D matrices (they differ at most in the sign of zero entries)
        assert torch.equal(T, R.heading_T([o["heading"] for o in obs]))
        assert set(got) == set(want)
        for k in want:
            if torch.is_tensor(want[k]):
                assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), k
            else:
                assert got[k] == want[k], k


def test_project_bev_ragged_lists_equal_padding(splat_cpu):
    from bevbert_b200.model.bev_utils import PointCloud
    pcl = PointCloud(np.radians(90), 1, 14, 14, 21, 0.5)
    clouds = [NB.node_cloud("v2_3", 0, t, 5, C=8, n=n) for t, n in enumerate((50, 1, 7))]
    pcs, nods, feats = (list(x) for x in zip(*clouds))
    bev, ob = pcl.project_bev(pcs, nods, feats)
    pad = torch.nn.utils.rnn.pad_sequence
    bev_p, ob_p = pcl.project_bev(pad(pcs, batch_first=True), pad(nods, batch_first=True, padding_value=True),
                                  pad(feats, batch_first=True))
    assert torch.equal(bev, bev_p) and torch.equal(ob, ob_p) and bev.shape == (3, 21, 21, 8)


# ------------------------------------------------------------------------------------------ C-level argument checks
class _Node(ctypes.Structure):
    _fields_ = [("pc", ctypes.c_void_p), ("no_depth", ctypes.c_void_p), ("feat", ctypes.c_void_p),
                ("n", ctypes.c_int64)]


def _call(nodes, offs, B, C=8, bf16=0, table=4096, S=64, T=128, bev=256, ob=512, D=21):
    from bevbert_b200 import _lib
    lib = _lib.load()
    arr = (_Node * max(len(nodes), 1))(*[_Node(*n) for n in nodes])
    o = (ctypes.c_int32 * len(offs))(*offs)
    rc = lib.bb_bev_splat_nodes(ctypes.addressof(arr) if nodes else None, len(nodes), o, B, table, S, T, C, bf16, D,
                                0.5, 0.5, bev, ob, None)
    return rc, (lib.bb_last_error() or b"").decode()


CASES = [
    (dict(nodes=[(16, 0, 32, 3)], offs=[0, 1], B=1, C=6), "C must be a positive multiple of 4"),
    (dict(nodes=[], offs=[0], B=-1), "must be >= 0"),
    (dict(nodes=[(16, 0, 32, 3)], offs=[0, 1], B=1, S=0), "null argument"),
    (dict(nodes=[(16, 0, 32, 3)], offs=[0, 1], B=1, bev=0), "null argument"),
    (dict(nodes=[(16, 0, 32, 3)], offs=[0, 1], B=1, table=0), "null argument"),
    (dict(nodes=[(0, 0, 32, 3)], offs=[0, 1], B=1), "null point or feature pointer"),
    (dict(nodes=[(16, 0, 32, 3), (16, 0, 48, 2)], offs=[0, 2, 1], B=2), "non-decreasing"),
    (dict(nodes=[(16, 0, 32, 3)], offs=[0, 2], B=1), "lie in [0, n_nodes]"),
    (dict(nodes=[(16, 0, 40, 3)], offs=[0, 1], B=1), "misaligned feature rows"),
    (dict(nodes=[(16, 0, 36, 3)], offs=[0, 1], B=1, bf16=1), "misaligned feature rows"),
    (dict(nodes=[(16, 0, 32, -1)], offs=[0, 1], B=1), "negative node size"),
    (dict(nodes=[], offs=[0], B=0), ""),
]


def test_c_entry_rejects_bad_arguments_before_any_launch():
    """Host arrays with fake device pointers, never dereferenced: every bad call returns its message, the empty batch
    returns 0.  The calls run in a process that sees no GPU, so a library that let one through could launch nothing."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys, json; sys.path[:0] = [sys.argv[1], sys.argv[1] + '/tests']; import test_nav_bev_cpu as t; "
            "print(json.dumps([t._call(**c) for c, _ in t.CASES]))")
    r = subprocess.run([sys.executable, "-c", code, root], env=dict(os.environ, CUDA_VISIBLE_DEVICES=""),
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    for (rc, msg), (case, want) in zip(json.loads(r.stdout.strip().splitlines()[-1]), CASES):
        if not want:
            assert rc == 0, (case, msg)
        else:
            assert rc != 0 and want in msg, (case, msg)
