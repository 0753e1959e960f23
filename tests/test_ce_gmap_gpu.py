"""GPU checks of the VLN-CE global-map image input (bb_ce_gmap_features / _bwd through graphs.install_ce_gmap_features):
15-step rollouts at B = 8 -> 5 -> 1 with the installed glue against the reference's torch glue around the same
panorama / navigation calls (bit-identical gmap_img_fts, fused_logits and actions), one call's gradient against the
reference's, parameter gradients of a teacher-forced loss, deterministic repeats, autocast, no_grad / frozen
embeddings, host synchronisations, other get_node_embeds callers, guards and rejections."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import ce_gmap_cases as C  # noqa: E402
from bevbert_b200 import _lib, ce_gmap, graphs  # noqa: E402
from oracle import ce_gmap_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def trainers(seed=3, merge_ghost=True):
    ref = C.Trainer(seed, DEV, merge_ghost)
    ins = C.Trainer(seed, DEV, merge_ghost)
    graphs.install_ce_gmap_features(ins)
    return ref, ins


class Recorder:
    """keeps every gmap_img_fts a trainer's _nav_gmap_variable returns"""

    def __init__(self, trainer):
        self.fts, inner = [], trainer._nav_gmap_variable

        def call(*a):
            out = inner(*a)
            self.fts.append(out["gmap_img_fts"].detach().clone())
            return out
        trainer._nav_gmap_variable = call


@pytest.mark.parametrize("merge_ghost", [True, False])
@pytest.mark.parametrize("train", [True, False])
def test_rollout_matches_reference(merge_ghost, train):
    ref, ins = trainers(merge_ghost=merge_ghost)
    rr, ri = Recorder(ref), Recorder(ins)
    with torch.set_grad_enabled(train):
        lr, ar, _ = C.rollout(ref, 11, train=train)
        li, ai, _ = C.rollout(ins, 11, train=train)
    assert len(rr.fts) == len(ri.fts) == len(C.SCHEDULE)
    for s, (a, b) in enumerate(zip(rr.fts, ri.fts)):
        assert a.shape == b.shape and a.dtype == b.dtype == torch.float32, s
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), s
    for s in range(len(C.SCHEDULE)):
        assert torch.equal(lr[s], li[s]) and np.array_equal(ar[s], ai[s]), s
    assert any(len(g.ghost_embeds) for g in ins.gmaps)


def test_installed_rollout_without_reference_glue():
    """update_graph's embedding arguments are not read: a rollout that passes None gets the same logits"""
    ref, ins = trainers()
    with torch.no_grad():
        lr, ar, _ = C.rollout(ref, 12, train=False)
        li, ai, _ = C.rollout(ins, 12, train=False, reference_glue=False)
    for s in range(len(C.SCHEDULE)):
        assert torch.equal(lr[s], li[s]) and np.array_equal(ar[s], ai[s]), s


def test_one_call_gradient_matches_reference():
    """within one navigation call every pano row gets at most a node part and a ghost part: the same values as
    torch's backward of the reference glue"""
    ref, ins = trainers()
    for t in (ref, ins):
        C.rollout(t, 13, schedule=[4] * 4, train=True)
    g = torch.randn(4, max(len(x.node_pos) + len(x.ghost_pos) for x in ref.gmaps) + 1, C.H, device=DEV)
    mem = ce_gmap.episode(ins.gmaps)
    _, rows = ce_gmap.trainer_method(lambda: C.Trainer._nav_gmap_variable(ins, None, None, None), ins.gmaps)
    fts = mem.features(rows)
    panos = [p for p, _, _ in mem.steps]
    got = torch.autograd.grad(fts, panos, g, allow_unused=True)
    # the reference on the same stored outputs
    rg = [R.GraphMap(False, 0.5, True, 0) for _ in range(4)]
    for x, y in zip(rg, ins.gmaps):
        x.node_pos, x.ghost_pos = y.node_pos, y.ghost_pos
    leaves = [p.detach().requires_grad_(True) for p in panos]
    for x, y in zip(rg, ins.gmaps):
        x.node_embeds = {vp: None for vp in y.node_embeds}
        x.ghost_embeds = {}
    for vp_map, y in zip(rg, ins.gmaps):
        for vp, h in y.node_embeds.items():
            p, _, m = mem.steps[h.s]
            vp_map.node_embeds[vp] = (torch.sum(leaves[h.s] * m.unsqueeze(2), 1) / torch.sum(m, 1, keepdim=True))[h.i]
        for vp, (h, n) in y.ghost_embeds.items():
            acc = None
            for s, i, k in h.terms:
                row = leaves[s][i][mem.steps[s][1][i] == 1][k]
                acc = row if acc is None else acc + row
            vp_map.ghost_embeds[vp] = [acc, n]
    want_fts = R.gmap_img_fts(rg)
    assert torch.equal(want_fts.view(torch.int32), fts.detach().view(torch.int32))
    want = torch.autograd.grad(want_fts, leaves, g, allow_unused=True)
    for s, (a, b) in enumerate(zip(got, want)):
        b = torch.zeros_like(a) if b is None else b
        assert torch.equal(a, b), s


def param_grads(trainer, seed):
    net = trainer.policy.net
    net.zero_grad(set_to_none=True)
    _, _, loss = C.rollout(trainer, seed, train=True)
    loss.backward()
    return {n: p.grad.clone() for n, p in net.named_parameters()}


def test_parameter_gradients_within_fp32_bound():
    ref, ins = trainers()
    gr, gi = param_grads(ref, 14), param_grads(ins, 14)
    for n in gr:
        err = float((gi[n].double() - gr[n].double()).norm() / gr[n].double().norm())
        assert err < 1e-5, (n, err)


def test_deterministic_repeats_bit_identical():
    _, ins = trainers()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a, b = param_grads(ins, 15), param_grads(ins, 15)
    finally:
        torch.use_deterministic_algorithms(prev)
    for n in a:
        assert torch.equal(a[n].view(torch.int32), b[n].view(torch.int32)), n


def test_autocast_changes_no_bit():
    _, ins = trainers()
    r = Recorder(ins)
    with torch.no_grad():
        C.rollout(ins, 16, train=False)
        base = list(r.fts)
        r.fts.clear()
        with torch.autocast("cuda", dtype=torch.float16):
            C.rollout(ins, 16, train=False)
    for a, b in zip(base, r.fts):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_no_grad_and_frozen_embeddings_record_nothing():
    _, ins = trainers()
    seen = []
    inner = ins._nav_gmap_variable
    ins._nav_gmap_variable = lambda *a: seen.append(inner(*a)) or seen[-1]
    with torch.no_grad():
        C.rollout(ins, 17, schedule=[3] * 3, train=False)
    ins.policy.net.scale.requires_grad_(False)
    ins.policy.net.bias.requires_grad_(False)
    C.rollout(ins, 17, schedule=[3] * 3, train=False)
    assert all(o["gmap_img_fts"].grad_fn is None and not o["gmap_img_fts"].requires_grad for o in seen)


def test_installed_glue_never_synchronises():
    _, ins = trainers()
    C.rollout(ins, 18, schedule=[4] * 3, train=True)      # warm: allocator, pinned pool, library
    rng = np.random.default_rng(0)
    inputs, ncand = C.step_inputs(rng, 4, DEV)
    cur_vp = [str(len(g.node_pos)) for g in ins.gmaps]
    cand_pos = [C.positions(rng, g, np.zeros(3), ncand[i]) for i, g in enumerate(ins.gmaps)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            ins.policy.net(mode="panorama", **inputs)
            for i, g in enumerate(ins.gmaps):
                g.update_graph(None, 4, cur_vp[i], np.zeros(3), None, ["c%d" % k for k in range(ncand[i])],
                               cand_pos[i], None, None)
            out = ins._nav_gmap_variable(cur_vp, None, None)
            out["gmap_img_fts"].sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    syncs = [str(x.message) for x in w if "synchroniz" in str(x.message).lower()]
    assert syncs == [], syncs


def test_get_node_embeds_for_other_callers():
    ref, ins = trainers()
    with torch.no_grad():
        C.rollout(ref, 19, schedule=[2] * 4, train=False)
        C.rollout(ins, 19, schedule=[2] * 4, train=False)
    for a, b in zip(ref.gmaps, ins.gmaps):
        for vp in list(a.node_pos) + list(a.ghost_pos):
            x, y = a.get_node_embeds(vp), b.get_node_embeds(vp)
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), vp


def test_unread_memory_poisoned_with_nan():
    """rows the map does not reference (environments without a node, padding views past every candidate) never reach
    gmap_img_fts, and both kernels write every element of their outputs: the output and gradient buffers come from
    freed NaN-filled blocks of the caching allocator"""
    mem = ce_gmap.Memory()
    pano = torch.full((3, 14, C.H), float("nan"), device=DEV)
    pano[1, :12] = torch.randn(12, C.H, device=DEV)
    nav = torch.zeros(3, 14, dtype=torch.int64, device=DEV)
    nav[1, 3] = nav[1, 7] = 1
    masks = torch.zeros(3, 14, dtype=torch.bool, device=DEV)
    masks[1, :12] = True
    pano[1, 12:] = 0      # masked views still enter torch's sum as x * 0, so they must be finite
    pano.requires_grad_(True)
    mem.record(pano, nav, masks)
    rows = [[ce_gmap.Node(mem, 0, 1), ce_gmap.Cands(mem, ((0, 1, 1), (0, 1, 0)))], []]
    torch.cuda.synchronize()
    poison = torch.full((2, 3, C.H), float("nan"), device=DEV)
    ptr = poison.data_ptr()
    del poison
    out = mem.features(rows)
    assert out.data_ptr() == ptr, "the output did not reuse the poisoned block"
    assert torch.isfinite(out).all()
    assert torch.equal(out[1], torch.zeros_like(out[1])) and torch.equal(out[0, 0], torch.zeros(C.H, device=DEV))
    want = (pano[1, 7] + pano[1, 3]).detach() / 2
    assert torch.equal(out[0, 2].view(torch.int32), want.view(torch.int32))
    gout = torch.randn_like(out)
    poison = torch.full_like(pano, float("nan"))
    ptr = poison.data_ptr()
    del poison
    got, = torch.autograd.grad(out, pano, gout)
    assert got.data_ptr() == ptr, "the gradient did not reuse the poisoned block"
    want = torch.zeros_like(got)
    want[1, :12] = gout[0, 1] / torch.tensor(12.0, device=DEV)
    want[1, 3] += gout[0, 2] * 0.5
    want[1, 7] += gout[0, 2] * 0.5
    assert torch.equal(got, want)
    # a candidate the row does not have gives NaN, loudly
    bad = mem.features([[ce_gmap.Cands(mem, ((0, 1, 2),))]])
    assert torch.isnan(bad[0, 1]).all()


def test_guards_and_rejections():
    mem = ce_gmap.Memory()
    pano = torch.zeros(2, 13, C.H, device=DEV)
    nav = torch.zeros(2, 13, dtype=torch.int64, device=DEV)
    masks = torch.ones(2, 13, dtype=torch.bool, device=DEV)
    with pytest.raises(TypeError):
        mem.record(pano.double(), nav, masks)
    with pytest.raises(ValueError):         # contiguous, but 4 bytes past a 16-byte boundary
        mem.record(torch.zeros(2 * 13 * C.H + 1, device=DEV)[1:].view(2, 13, C.H), nav, masks)
    with pytest.raises(TypeError):
        mem.record(pano.transpose(0, 1), nav, masks)
    with pytest.raises(TypeError):
        mem.record(pano, nav.int(), masks)
    with pytest.raises(TypeError):
        mem.record(pano, nav, masks.float())
    with pytest.raises(ValueError):
        mem.record(torch.zeros(2, 64, C.H, device=DEV), torch.zeros(2, 64, dtype=torch.int64, device=DEV),
                   torch.ones(2, 64, dtype=torch.bool, device=DEV))
    mem.record(pano, nav, masks)
    with pytest.raises(ValueError):
        mem.record(torch.zeros(2, 13, 512, device=DEV), nav, masks)
    with pytest.raises(ValueError):
        ce_gmap.Cands(mem, ((0, 0, 0),)) / 2
    with pytest.raises(ValueError):
        mem.features([[ce_gmap.Node(ce_gmap.Memory(), 0, 0)]])
    lib = _lib.load()
    out = torch.zeros(1, 2, C.H, device=DEV)
    t = torch.zeros(64, dtype=torch.int32, device=DEV)
    assert lib.bb_ce_gmap_features(t.data_ptr(), 0, 1, 2, 766, out.data_ptr(), None) != 0
    assert lib.bb_ce_gmap_features(None, 0, 1, 2, C.H, out.data_ptr(), None) != 0
    assert lib.bb_ce_gmap_features(t.data_ptr(), 0, 0, 2, C.H, out.data_ptr(), None) != 0
    assert lib.bb_ce_gmap_features(t.data_ptr(), 0, 1, 2, C.H, out.data_ptr() + 4, None) != 0
    assert lib.bb_ce_gmap_features_bwd(t.data_ptr(), 0, 1, 13, 2, C.H, out.data_ptr(), None) != 0
    assert lib.bb_ce_gmap_features_bwd(t.data_ptr(), 1, 0, 13, 2, C.H, out.data_ptr(), None) == 0
    # update_graph without this step's panorama call
    _, ins = trainers()
    ins.gmaps = [R.GraphMap(False, 0.5, True, 0)]
    ce_gmap.attach(ins, ins.gmaps[0], ce_gmap.Memory())
    with pytest.raises(RuntimeError):
        ins.gmaps[0].update_graph(None, 1, "0", np.zeros(3), None, [], [], None, None)
    ins.gmaps.append(R.GraphMap(False, 0.5, True, 0))
    with pytest.raises(RuntimeError):
        ins._nav_gmap_variable(["0", "0"], None, None)
