"""bb_bev_splat_nodes on the GPU: the agent-side BEV pooled straight from node point clouds, bit for bit against the
CPU oracle (tests/nav_bev_oracle.py nav_splat_nodes) and the eager chain it replaces, with shared nodes, views into a
batched PointCloud.forward output, samples above the old 51,200-point limit, NaN everywhere the kernel must not read,
guard regions, the agent adapter feeding the navigation call, repeatability and argument checks."""
import math

import numpy as np
import pytest
import torch

import nav_bev_cases as NB
import nav_bev_oracle as R

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
D, RES = 21, 0.5


@pytest.fixture(scope="module")
def K():
    from bevbert_b200 import bev_nodes
    assert torch.cuda.is_available()
    return bev_nodes


def _pool(C, dtype, n_big=24):
    """Node clouds on the GPU: n_big nodes of 2352 points as views into one batched PointCloud.forward output (the
    agents' lift), plus nodes of 1 and 7 points; node 'edge' holds hand-placed points (exact .5 cell edges in the
    identity frame, y == clip, outside the map, NaN)."""
    from bevbert_b200.model.bev_utils import PointCloud
    pcl = PointCloud(math.radians(90), 1, 14, 14, D, RES)
    bs = n_big
    depth = NB.synth.det_uniform((bs * 12, 1, 14, 14), 3, 1, 0.0, 0.6)
    depth[depth < 0.03] = 0.0
    heads = torch.arange(bs * 12, dtype=torch.float64) * (math.pi / 6)
    T = torch.zeros(bs * 12, 4, 4)
    T[:, 0, 0], T[:, 0, 2], T[:, 1, 1], T[:, 2, 0], T[:, 2, 2], T[:, 3, 3] = (
        heads.cos().float(), heads.sin().float(), -1.0, -heads.sin().float(), heads.cos().float(), 1.0)
    T[:, 0, 3] = NB.synth.det_uniform((bs * 12,), 3, 2, -2.0, 2.0)
    T[:, 1, 3] = 1.25
    pc, nod = pcl.forward(depth.cuda() * 10, T.cuda())
    pc, nod = pc.reshape(bs, -1, 3), nod.reshape(bs, -1)
    feat = NB.synth.det_uniform((bs, 2352, C), 3, 4, -1.7, 1.7).to(dtype).cuda()
    nodes = [(pc[i], nod[i], feat[i]) for i in range(bs)]
    for s, n in enumerate((1, 7, 1, 7, 1)):
        p, m, f = NB.node_cloud("v3_3", 9, s, 7, C=C, n=n, feat_dtype=dtype)
        nodes.append((p.cuda(), m.cuda(), f.cuda()))
    edge = torch.tensor([[0.25, 0.0, 0.75], [-0.25, 0.5, 1.25], [5.25, 0.0, -5.25], [5.26, 0.0, 0.0],
                         [-5.25, 0.2, 5.24], [0.0, 0.5000001, 0.0], [float("nan"), 0.0, 0.0], [0.0, 0.0, float("nan")],
                         [0.75, 0.5, -0.25], [2.25, -0.3, 3.75]])
    fe = NB.synth.det_uniform((edge.shape[0], C), 8, 1, -1.0, 1.0).to(dtype)
    nodes.append((edge.cuda(), torch.zeros(edge.shape[0], dtype=torch.bool).cuda(), fe.cuda()))
    return nodes


def _frames(B, seed):
    """per sample: identity (exact edges), the agents' heading-only frame, or a general rotation + translation"""
    from bevbert_b200.agent_bev import ego_frames
    S = torch.zeros(B, 3)
    T = torch.eye(4).repeat(B, 1, 1)
    for b in range(B):
        if b % 3 == 1:
            s, t = ego_frames([{"position": [0.3 * b, -1.1, 1.5], "heading": 0.7 * b - 2.0}])
            S[b], T[b] = torch.from_numpy(s[0]), torch.from_numpy(t[0])
        elif b % 3 == 2:
            q, _ = torch.linalg.qr(NB.synth.det_uniform((3, 3), seed, b, -1.0, 1.0).double())
            T[b, :3, :3] = q.float()
            T[b, :3, 3] = NB.synth.det_uniform((3,), seed, 100 + b, -0.5, 0.5)
            S[b] = NB.synth.det_uniform((3,), seed, 200 + b, -2.0, 2.0)
    return S.cuda(), T.cuda()


def _selection(B, n_pool):
    """0..30 nodes per sample, different per sample, nodes shared between samples; sample 1 (if any) holds 23 big
    nodes (54,096 points, above the old 51,200-point limit)"""
    counts = [0, 23, 5, 30, 1, 12, 2, 7, 19, 3, 0, 9, 26, 4, 11, 6]
    sel = []
    for b in range(B):
        c = counts[b % len(counts)] if B > 1 else 8
        if c == 23:
            sel.append(list(range(23)))
        else:
            sel.append([(7 * b + 5 * j) % n_pool for j in range(c)])
    sel[-1] = sel[-1] + [n_pool - 1]     # the edge node, in a sample with the identity frame
    return sel


CASES = [(1, torch.float32, 768), (4, BF, 772), (4, torch.float32, 772), (16, torch.float32, 4), (16, BF, 768)]


@pytest.mark.parametrize("B,dtype,C", CASES)
def test_kernel_equals_oracle_bit_for_bit(K, B, dtype, C):
    pool = _pool(C, dtype)
    sel = _selection(B, len(pool))
    clouds = [[pool[j] for j in s] for s in sel]
    S, T = _frames(B, seed=B)
    bev, ob = K.bev_splat_nodes(clouds, S, T, D, RES)
    rb, rob = R.nav_splat_nodes(clouds, S.cpu(), T.cpu(), D, RES)
    assert torch.equal(bev.cpu(), rb), float((bev.cpu() - rb).abs().nan_to_num().max())
    assert torch.equal(ob.cpu(), rob)
    if B > 1:
        assert sum(pool[j][0].shape[0] for j in sel[1]) > 51200
    assert (~rob).any() and rob.any()


def test_project_bev_ragged_list_equals_padded(K):
    from bevbert_b200.model.bev_utils import PointCloud
    pcl = PointCloud(math.radians(90), 1, 14, 14, D, RES)
    pool = _pool(768, torch.float32, n_big=3)
    pcs, nods, feats = (list(x) for x in zip(*pool[:3], pool[4], pool[-1]))
    bev, ob = pcl.project_bev(pcs, nods, feats)
    pad = torch.nn.utils.rnn.pad_sequence
    bp, obp = pcl.project_bev(pad(pcs, batch_first=True), pad(nods, batch_first=True, padding_value=True),
                              pad(feats, batch_first=True))
    assert torch.equal(bev, bp) and torch.equal(ob, obp)


def _eager_chain(clouds, S, T, pcl):
    """gather (torch.cat) -> pad_sequence -> fixed-order ego transform -> project_bev, all on the GPU"""
    pad = torch.nn.utils.rnn.pad_sequence
    pc = pad([torch.cat([n[0] for n in c]) for c in clouds], batch_first=True)
    nod = pad([torch.cat([n[1] for n in c]) for c in clouds], batch_first=True, padding_value=True)
    ft = pad([torch.cat([n[2] for n in c]) for c in clouds], batch_first=True)
    p = pc - S[:, None, :]
    e = []
    for j in range(3):
        acc = p[..., 0] * T[:, None, j, 0]
        acc = acc + p[..., 1] * T[:, None, j, 1]
        acc = acc + p[..., 2] * T[:, None, j, 2]
        acc = acc + T[:, None, j, 3]
        e.append(acc)
    bev, ob = pcl.project_bev(torch.stack(e, -1), nod, ft)
    return bev.reshape(len(clouds), -1, bev.shape[-1]), ob


@pytest.mark.parametrize("dtype", [torch.float32, BF])
def test_splat_nodes_equals_eager_chain(K, dtype):
    from bevbert_b200.model.bev_utils import PointCloud
    pcl = PointCloud(math.radians(90), 1, 14, 14, D, RES)
    pool = _pool(768, dtype, n_big=8)
    B = 4
    clouds = [[pool[j] for j in s] for s in ([0, 1, 2], [3, 8, 4, 5, 6, 7], [2], [9, 10, 0, 13])]
    S, T = _frames(B, seed=3)
    bev, ob = pcl.splat_nodes(clouds, S, T)
    be, obe = _eager_chain(clouds, S, T, pcl)
    assert torch.equal(bev, be) and torch.equal(ob, obe)


def test_reads_and_writes_stay_in_bounds(K):
    """Direct C call on hand-built buffers: NaN in the feature rows of every dropped point and in every batch row no
    node refers to, outputs inside NaN / 0xAB guard regions that must come back untouched."""
    from bevbert_b200 import _lib
    C, B, G = 772, 3, 4096
    pool = _pool(C, torch.float32, n_big=6)
    sel = [[0, 24 - 18, 2], [], [3, 1, len(pool) - 1, 6]]
    sel = [[min(j, len(pool) - 1) for j in s] for s in sel]
    S, T = _frames(B, seed=5)
    clouds = [[pool[j] for j in s] for s in sel]
    for b, nodes in enumerate(clouds):                # features of dropped points -> NaN (every use of the node)
        for node in nodes:
            keep = torch.zeros(node[0].shape[0], dtype=torch.bool)
            for bb, nn_ in enumerate(clouds):
                for other in nn_:
                    if other[0].data_ptr() == node[0].data_ptr():
                        idx, _ = R.nav_cell_index([other], S[bb].cpu(), T[bb].cpu(), D, RES)
                        keep |= idx >= 0
            node[2][~keep.cuda()] = float("nan")
    used = {pool[j][2].data_ptr() for s in sel for j in s}
    for p_ in pool[:6]:                                 # batch rows of the forward output no sample gathers
        if p_[2].data_ptr() not in used:
            p_[2].fill_(float("nan"))
    rb, rob = R.nav_splat_nodes(clouds, S.cpu(), T.cpu(), D, RES)
    bev_buf = torch.full((G + B * D * D * C + G,), float("nan"), device="cuda")
    ob_buf = torch.full((G + B * D * D + G,), 0xAB, dtype=torch.uint8, device="cuda")
    rows = [(n[0].data_ptr(), n[1].data_ptr(), n[2].data_ptr(), n[0].shape[0]) for c in clouds for n in c]
    offs = np.cumsum([0] + [len(c) for c in clouds]).astype(np.int32)
    host = np.array(rows, dtype=np.int64)
    table = torch.empty(32 * len(rows) + 4 * (B + 1), dtype=torch.uint8, device="cuda")
    lib = _lib.load()
    rc = lib.bb_bev_splat_nodes(host.ctypes.data, len(rows), offs.ctypes.data, B, table.data_ptr(), S.data_ptr(),
                                T.data_ptr(), C, 0, D, RES, 0.5, bev_buf.data_ptr() + 4 * G, ob_buf.data_ptr() + G,
                                torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "bb_bev_splat_nodes")
    torch.cuda.synchronize()
    assert torch.isnan(bev_buf[:G]).all() and torch.isnan(bev_buf[-G:]).all()
    assert (ob_buf[:G] == 0xAB).all() and (ob_buf[-G:] == 0xAB).all()
    got = bev_buf[G:-G].view(B, D * D, C).cpu()
    assert torch.equal(got, rb) and not torch.isnan(got).any()
    assert torch.equal(ob_buf[G:-G].view(B, D * D).cpu().bool(), rob)
    assert not rob[1].any() and (got[1] == 0).all()      # the sample without nodes


def test_launch_table_layout(K):
    """the rows the wrapper uploads: (points, mask, features, n) per node in sample order, then the B+1 offsets"""
    pool = _pool(8, torch.float32, n_big=2)
    clouds = [[pool[0], pool[3]], [], [pool[3], pool[1], pool[-1]]]
    S, T = _frames(3, seed=1)
    K.bev_splat_nodes(clouds, S, T, D, RES)
    torch.cuda.synchronize()
    slot = K._NODE_SLOTS[K._NODE_TURN[0] ^ 1]
    dev = slot.dev.cpu().numpy()
    rows = dev[:32 * 5].view(np.int64).reshape(5, 4)
    want = [(n[0].data_ptr(), n[1].data_ptr(), n[2].data_ptr(), n[0].shape[0]) for c in clouds for n in c]
    assert [tuple(r) for r in rows.tolist()] == want
    assert dev[32 * 5:32 * 5 + 16].view(np.int32).tolist() == [0, 2, 2, 5]


def test_repeatable_and_deterministic_mode(K):
    pool = _pool(768, BF, n_big=6)
    clouds = [[pool[j] for j in s] for s in ([0, 1, 2, 3], [5, 4, 11], [2, 0])]
    S, T = _frames(3, seed=2)
    a = K.bev_splat_nodes(clouds, S, T, D, RES)
    b = K.bev_splat_nodes(clouds, S, T, D, RES)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        c = K.bev_splat_nodes(clouds, S, T, D, RES)
    finally:
        torch.use_deterministic_algorithms(prev)
    for x in (b, c):
        assert torch.equal(a[0], x[0]) and torch.equal(a[1], x[1])


def test_adapter_equals_oracle_and_feeds_navigation(K):
    """nav_bev_variable on stub agents equals the oracle's _nav_bev_variable; the navigation call fed by its dict equals
    the call fed by the eager chain's dict, eagerly and through GraphedNavigation."""
    from bevbert_b200.agent_bev import nav_bev_variable
    from bevbert_b200.graphs import GraphedNavigation
    from test_nav_graphs_gpu import _inputs, _model
    B, Dn = 3, 11
    model = _model(0)
    graphed = GraphedNavigation(model)
    last = None
    for obs, gmaps, order in NB.run_stub_episode(B=B, steps=24, device="cuda"):
        agent = NB.StubAgent(B, D=Dn, res=1.0, pc_order=order, device="cuda")
        got = nav_bev_variable(agent, obs, gmaps)
        cpu_maps = [NB.StubGraphMap(g.start_vp, g.graph) for g in gmaps]
        for g, cg in zip(gmaps, cpu_maps):
            cg.node_pc = {k: [t.cpu() for t in v] for k, v in g.node_pc.items()}
        want = R.nav_bev_variable(obs, cpu_maps, order, Dn, 1.0, agent._map_cand_to_bev, agent.bev_pos)
        for k in want:
            if torch.is_tensor(want[k]):
                assert torch.equal(got[k].cpu(), want[k]), (k, order)
            else:
                assert got[k] == want[k]
        last = (obs, gmaps, order, agent, got)
    obs, gmaps, order, agent, got = last
    from bevbert_b200.model.bev_utils import PointCloud
    pcl = PointCloud(math.radians(90), 1, 14, 14, Dn, 1.0)
    clouds = [[g.node_pc[c] for c in R.gather_nodes(g, ob["viewpoint"], order)] for ob, g in zip(obs, gmaps)]
    from bevbert_b200.agent_bev import ego_frames
    s, t = ego_frames(obs)
    eager_bev, _ = _eager_chain(clouds, torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda(), pcl)
    assert torch.equal(eager_bev, got["bev_fts"])
    lang, pano, nav = _inputs(B, 8, 4, D=Dn)
    outs = []
    with torch.no_grad():
        t_emb = model("language", lang)
        for bev in (got["bev_fts"], eager_bev):
            nb = dict(nav, txt_embeds=t_emb, bev_fts=bev, bev_pos_fts=got["bev_pos_fts"], bev_masks=got["bev_masks"])
            outs.append((model("navigation", nb), graphed("navigation", nb)))
    for k in ("gmap_embeds", "global_logits", "local_logits", "fused_logits"):
        assert torch.equal(outs[0][0][k], outs[1][0][k]) and torch.equal(outs[0][1][k], outs[1][1][k]), k


def test_argument_checks(K):
    from bevbert_b200._lib import BevbertLibraryError
    pool = _pool(8, torch.float32, n_big=2)
    S, T = _frames(2, seed=1)
    ok = [[pool[0]], [pool[1]]]
    p, m, f = pool[0]
    bad = [
        ([[(p.cpu(), m.cpu(), f.cpu())], [pool[1]]], RuntimeError, "must be a CUDA tensor"),
        ([[(p, m, f.cpu())], [pool[1]]], RuntimeError, "must be a CUDA tensor"),
        ([[(p.double(), m, f)], [pool[1]]], TypeError, "points must be torch.float32"),
        ([[(p, m.float(), f)], [pool[1]]], TypeError, "no-depth mask"),
        ([[(p, m, f.half())], [pool[1]]], TypeError, "features must be float32 or bfloat16"),
        ([[(p, m, f.to(BF))], [pool[1]]], TypeError, "like the other nodes"),
        ([[(p, m, torch.cat([f, f], 1))], [pool[1]]], ValueError, "feature columns"),
        ([[(p, m, torch.cat([f, f], 1)[:, ::2])], [pool[1]]], ValueError, "must be contiguous"),
        ([[(p[:, :2].contiguous(), m, f)], [pool[1]]], ValueError, "expected points"),
        ([[], []], ValueError, "pass C"),
    ]
    for clouds, exc, msg in bad:
        with pytest.raises(exc, match=msg):
            K.bev_splat_nodes(clouds, S, T, D, RES)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        K.bev_splat_nodes(ok, S.cpu(), T, D, RES)
    with pytest.raises(ValueError, match="S_w2c must be"):
        K.bev_splat_nodes(ok, S[:1], T, D, RES)
    with pytest.raises(BevbertLibraryError, match="C must be a positive multiple of 4"):
        K.bev_splat_nodes([[(p, m, f[:, :6].contiguous())], []], S, T, D, RES)
    with pytest.raises(BevbertLibraryError, match="misaligned feature rows"):
        fo = torch.empty(f.numel() + 1, device="cuda")[1:].view_as(f)
        K.bev_splat_nodes([[(p, m, fo)], []], S, T, D, RES)
    e, eo = K.bev_splat_nodes([[], []], S, T, D, RES, C=8)
    assert (e == 0).all() and not eo.any()
