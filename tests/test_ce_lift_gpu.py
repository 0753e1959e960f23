"""GPU checks of the VLN-CE trainer's lift on the kernels: bb_bev_lift_points bit for bit against the fixed-order oracle
(tests/ce_lift_oracle.py), canary bytes around its outputs, bb_bev_lift_index unchanged by the shared camera-to-world
function, the installed lift against the reference's torch chain on the device (cuBLAS bmm), and a 15-step episode
with the installed waypoint step feeding the lift, the BEV and the navigation call."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [p for p in (ROOT, os.path.join(ROOT, "tests")) if p not in sys.path]

import ce_lift_cases as C  # noqa: E402
import ce_lift_oracle as O  # noqa: E402
from bevbert_b200 import agent_bev, bev_nodes, graphs  # noqa: E402
from bevbert_b200 import kernels as K  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "small_ce_lift.pt"), weights_only=False)


def bits(x):
    return x.detach().contiguous().view(torch.int32)


def ulps(a, b):
    def key(x):
        i = bits(x).to(torch.int64)
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)
    return (key(a) - key(b)).abs()


def random_case(B, seed):
    rng = np.random.default_rng(seed)
    pos = [rng.uniform(-50, 50, 3) for _ in range(B)]
    heads = [float(rng.uniform(0, 2 * math.pi)) for _ in range(B)]
    return pos, heads, C.depth_grid(rng, B)


def kernel_lift(pos, heads, depth, shift):
    T = torch.from_numpy(agent_bev.lift_frames(pos, heads)).to(DEV)
    fx, fy, cx, cy = agent_bev.lift_intrinsics(C.Projector("cpu"))
    return bev_nodes.bev_lift_points(depth.to(DEV).reshape(-1, 14, 14), T, shift.to(DEV), 10.0, fx, fy, cx, cy)


@pytest.mark.parametrize("B", [1, 5, 8])
def test_lift_points_equals_oracle(B):
    for seed, shift in ((B, torch.zeros(3)), (B + 100, torch.tensor([0.25, -1.5, 3.0]))):
        pos, heads, depth = random_case(B, seed)
        pts, nod = kernel_lift(pos, heads, depth, shift)
        o = O.lift(pos, heads, depth, shift)
        assert torch.equal(bits(pts.reshape(B, -1, 3).cpu()), bits(o["pc"]))
        assert torch.equal(nod.reshape(B, -1).cpu(), o["pc_mask"])


def test_lift_points_golden_cases():
    for g in GOLD["cases"]:
        pos, _, depth, shift, _ = C.case_inputs(g["case"])
        pts, nod = kernel_lift(pos, g["headings"], depth, shift)
        B = g["case"]["B"]
        o = O.lift(pos, g["headings"], depth, shift)
        assert torch.equal(bits(pts.reshape(B, -1, 3).cpu()), bits(o["pc"]))
        assert torch.equal(nod.reshape(B, -1).cpu(), g["pc_mask"])


@pytest.mark.parametrize("N", [1, 7, 131])       # 196 N points: never a multiple of the 256-thread block
def test_lift_points_odd_sizes_and_canaries(N):
    g = torch.Generator().manual_seed(N)
    depth = torch.rand(N, 14, 14, generator=g)
    depth[:, ::3, 1::2] = 0.0
    T = torch.randn(N, 4, 4, generator=g)
    shift = torch.randn(3, generator=g)
    n, pad = N * 196, 64
    pbuf = torch.full((n * 3 + 2 * pad,), -7.25, device=DEV)
    mbuf = torch.full((n + 2 * pad,), 0xA5, dtype=torch.uint8, device=DEV)
    lib = K._lib.load()
    fx, fy, cx, cy = agent_bev.lift_intrinsics(C.Projector("cpu"))
    dd, Td, sd = depth.to(DEV), T.to(DEV), shift.to(DEV)
    K._lib.check(lib.bb_bev_lift_points(dd.data_ptr(), Td.data_ptr(), N, 14, 14, 10.0, fx, fy, cx, cy, sd.data_ptr(),
                                        pbuf[pad:].data_ptr(), mbuf[pad:].data_ptr(), K._stream()), "lift_points")
    pb, mb = pbuf.cpu(), mbuf.cpu()
    assert (pb[:pad] == -7.25).all() and (pb[pad + 3 * n:] == -7.25).all()
    assert (mb[:pad] == 0xA5).all() and (mb[pad + n:] == 0xA5).all()
    xyz1, mask = O.camera_xyz1(depth)
    assert torch.equal(bits(pb[pad:pad + 3 * n].view(N, 196, 3)), bits(O.world_points(xyz1, T, shift)))
    assert torch.equal(mb[pad:pad + n].view(N, 196).bool(), mask)


def test_lift_points_rejections():
    lib = K._lib.load()
    d = torch.zeros(2, 14, 14, device=DEV)
    T = torch.zeros(2, 4, 4, device=DEV)
    s = torch.zeros(4, device=DEV)
    p = torch.zeros(2 * 196 * 3 + 1, device=DEV)
    m = torch.zeros(2 * 196, dtype=torch.uint8, device=DEV)
    good = [d.data_ptr(), T.data_ptr(), 2, 14, 14, 10.0, 7.0, 7.0, 7.0, 7.0, s.data_ptr(), p.data_ptr(), m.data_ptr(),
            K._stream()]
    assert lib.bb_bev_lift_points(*good) == 0
    for i, v in ((0, 0), (1, 0), (10, 0), (11, 0), (12, 0), (0, d.data_ptr() + 2), (11, p.data_ptr() + 1),
                 (10, s.data_ptr() + 2), (2, 0), (2, -1), (3, 0), (4, -14)):
        args = list(good)
        args[i] = v
        assert lib.bb_bev_lift_points(*args) != 0, (i, v)
    # sizes the launch cannot index, rejected before anything is written
    for N, Hf, Wf in ((2, 1 << 16, 1 << 16), (1 << 30, 1024, 1024)):
        args = list(good)
        args[2:5] = N, Hf, Wf
        assert lib.bb_bev_lift_points(*args) != 0, (N, Hf, Wf)


def test_lift_index_still_equals_oracle():
    from oracle import bevbert_ref as R
    g = torch.Generator().manual_seed(5)
    depths = torch.rand(3, 12, 14, 14, generator=g)
    depths[:, :, ::4] = 0.0
    T_c2w = torch.randn(3, 12, 4, 4, generator=g)
    S = torch.randn(3, 3, generator=g)
    Tw = torch.randn(3, 4, 4, generator=g)
    idx, pc = K.bev_lift_index(depths.to(DEV), T_c2w.to(DEV), S.to(DEV), Tw.to(DEV), 21, 0.5, want_pc=True)
    rpc, nod = R.lift_points(depths, T_c2w, S, Tw)
    assert torch.equal(bits(pc.cpu()), bits(rpc.reshape(pc.shape)))
    assert torch.equal(idx.cpu().long(), R.cell_index(rpc, nod, 21, 0.5).reshape(idx.shape))


# ----------------------------------------------------------------- the installed lift against the reference's chain
def reference_lift(trainer, cur_pos, cur_ori, rgb_grid, depth_grid):
    """lift (ss_trainer_BEV.py:386-410) and PointCloud.forward (bev_utils.py:349-378) as torch runs them on the device"""
    h = agent_bev._trainer_heading_fn(trainer)
    bs = len(cur_pos)
    T = O.lift_T(cur_pos, [h(o) for o in cur_ori]).cuda()
    depth = (depth_grid.reshape(-1, 1, 14, 14).cuda() * 10)[:, 0, :, :]
    no_depth_mask = depth == 0
    fx, fy, cx, cy = (v.cuda() for v in O.intrinsics())
    N = depth.shape[0]
    x_rows = torch.arange(14, device=DEV).unsqueeze(0).repeat((14, 1)).unsqueeze(0).repeat((N, 1, 1)).float()
    y_cols = torch.arange(14, device=DEV).unsqueeze(1).repeat((1, 14)).unsqueeze(0).repeat((N, 1, 1)).float()
    x_scale, y_scale = (x_rows + 0.5 - cx) / fx, (y_cols + 0.5 - cy) / fy
    z = depth / float(1.0)
    xyz1 = torch.cat(((z * x_scale).unsqueeze(3), (z * y_scale).unsqueeze(3), z.unsqueeze(3),
                      torch.ones((N, 14, 14), device=DEV).unsqueeze(3)), dim=3)
    xyz1 = torch.reshape(xyz1, (N, 196, 4))
    world = torch.bmm(T, torch.transpose(xyz1, 1, 2)).transpose(1, 2)[:, :, :3]
    world -= trainer.projector.world_shift_origin
    pc = world.reshape(N, 14, 14, 3)
    return pc.reshape(bs, -1, 3), no_depth_mask.reshape(bs, -1), rgb_grid.reshape(-1, 14, 14, 768).reshape(bs, -1, 768)


def bev_of(trainer, vps, pos, ori, clouds, prev=None):
    """stores each environment's cloud at a new node vps[i], linked to its previous node prev[i] (vp, pos) if any"""
    for i, gm in enumerate(trainer.gmaps):
        gm.visit(vps[i], pos[i], [prev[i]] if prev and prev[i] else [], clouds[i])
    return agent_bev.ce_nav_bev_variable(trainer, vps, pos, ori)


def test_installed_lift_against_device_chain():
    worst, n = 0, 0
    for g in GOLD["cases"]:
        B = g["case"]["B"]
        pos, ori, depth, _, _ = C.case_inputs(g["case"])
        ins, ref = C.LiftTrainer(B, DEV, g["case"]["shift"]), C.LiftTrainer(B, DEV, g["case"]["shift"])
        graphs.install_ce_lift(ins)
        rgb = C.rgb_grid(B, DEV)
        d = depth.to(DEV)
        got, want = ins.lift(pos, ori, rgb, d), reference_lift(ref, pos, ori, rgb, d)
        assert got[0].shape == want[0].shape and torch.equal(got[1], want[1])
        assert got[2].data_ptr() == rgb.data_ptr() and got[2].shape == (B, 2352, 768)
        u = ulps(got[0], want[0])
        worst, n = max(worst, int(u.max())), n + int((u > 0).sum())
        vps = ["n0"] * B
        a = bev_of(ins, vps, [tuple(p) for p in pos], ori, [tuple(t[i] for t in got) for i in range(B)])
        b = bev_of(ref, vps, [tuple(p) for p in pos], ori, [tuple(t[i] for t in want) for i in range(B)])
        for k in ("bev_fts", "bev_pos_fts", "bev_masks", "bev_nav_masks", "bev_cand_idxs"):
            assert torch.equal(a[k], b[k]), k
    print("installed lift vs cuBLAS bmm chain: %s (largest difference %d ulp, %d coordinates differ)"
          % ("bit-identical" if worst == 0 else "not bit-identical", worst, n))


# ------------------------------------------------------------------------------------------ a whole 15-step episode
def test_episode_with_installed_waypoint_step():
    import ce_nav_cases as NC
    import ce_waypoint_step_cases as WC
    from bevbert_b200 import synth
    from bevbert_b200.model.ce_nav import GlocalTextPathNavCMT
    net, wp = WC.Net(31, DEV), WC.predictor(31, DEV)
    graphs.install_ce_waypoint_step(net)
    nav = synth.det_init_(GlocalTextPathNavCMT(NC.config()), seed=NC.WEIGHT_SEED).to(DEV).eval()
    schedule = [8] * 5 + [5] * 5 + [1] * 5
    ins, ref = C.LiftTrainer(8, DEV), C.LiftTrainer(8, DEV)
    graphs.install_ce_lift(ins)
    rng = np.random.default_rng(7)
    pos = [tuple(rng.uniform(-20, 20, 3)) for _ in range(8)]
    ori = [C.quaternion_at(float(rng.uniform(0, 2 * math.pi))) for _ in range(8)]
    prev = [None] * 8
    with torch.no_grad():
        lang = {k: v.to(DEV) for k, v in NC.lang_inputs(8).items()}
        txt = nav.forward_txt(lang["txt_ids"], lang["txt_masks"])
        for stepk, B in enumerate(schedule):
            while len(pos) > B:                      # a middle environment's episode ends
                j = len(pos) // 2
                for lst in (pos, ori, prev, ins.gmaps, ref.gmaps):
                    lst.pop(j)
                txt = torch.cat([txt[:j], txt[j + 1:]])
                lang = {k: torch.cat([v[:j], v[j + 1:]]) for k, v in lang.items()}
            out = net(mode="waypoint", waypoint_predictor=wp, observations=WC.observations(B, 300 + stepk, DEV),
                      in_train=False)
            rgb, depth = out["pano_rgb_grid"], out["pano_depth_grid"]
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                got = ins.lift(pos, ori, rgb, depth)
            finally:
                torch.cuda.set_sync_debug_mode("default")
            want = reference_lift(ref, pos, ori, rgb, depth)
            assert torch.equal(got[1], want[1])
            vps = ["s%d" % stepk] * B                 # identify_node makes a fresh node every step
            a = bev_of(ins, vps, pos, ori, [tuple(t[i] for t in got) for i in range(B)], prev)
            b = bev_of(ref, vps, pos, ori, [tuple(t[i] for t in want) for i in range(B)], prev)
            assert torch.equal(a["bev_fts"], b["bev_fts"])
            prev = [(vps[i], pos[i]) for i in range(B)]
            logits, acts = [], []
            for bev in (a, b):
                inp = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in NC.nav_inputs(B, step=stepk).items()}
                inp["bev_fts"] = bev["bev_fts"]
                inp["gmap_img_fts"] = torch.ones(B, inp["gmap_masks"].shape[1], 768, device=DEV) * 0.01
                inp["txt_embeds"], inp["txt_masks"] = txt, lang["txt_masks"]
                o = nav.forward_navigation(*[inp[k] for k in NC.NAV_ARGS])["fused_logits"]
                logits.append(o)
                acts.append(o.argmax(-1).cpu().numpy())
            assert torch.equal(bits(logits[0]), bits(logits[1])) and np.array_equal(acts[0], acts[1]), stepk
            for i in range(B):
                pos[i] = tuple(np.add(pos[i], [0.5 * (int(acts[0][i]) % 3 - 1), 0.0, -0.4]))
                ori[i] = C.quaternion_at(0.7 * stepk + 0.3 * i)


def test_heading_frames_zero_signs_change_no_ego_point():
    """heading_frames now carries transfrom3D's signed zeros in T[0,1], T[1,2], T[2,1]; the ego transform ends each row
    with + T[j,3] = +0, so every ego point (zero coordinates included) is bit-identical to the +0-entry frames'"""
    h = np.array([0.3, -1.2, 2.5, 4.0, math.pi, -0.0])
    _, T = agent_bev.heading_frames(np.zeros((len(h), 3)), h)
    old = T.copy()
    old[:, 0, 1] = old[:, 1, 2] = old[:, 2, 1] = 0.0
    assert (np.signbit(T) != np.signbit(old)).any()
    g = torch.Generator().manual_seed(11)
    depths = torch.rand(len(h), 12, 14, 14, generator=g)
    depths[:, :, ::2] = 0.0                                      # these pixels land exactly on the origin
    T_c2w = torch.randn(len(h), 12, 4, 4, generator=g)
    T_c2w[..., :3, 3] = 0.0
    S = torch.zeros(len(h), 3)
    out = [K.bev_lift_index(depths.to(DEV), T_c2w.to(DEV), S.to(DEV), torch.from_numpy(t).to(DEV), 11, 1.0,
                            want_pc=True) for t in (T, old)]
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(bits(out[0][1]), bits(out[1][1]))
