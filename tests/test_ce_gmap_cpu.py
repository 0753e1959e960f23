"""CPU checks of the VLN-CE global-map image glue (oracle/ce_gmap_ref.py, the host half of bevbert_b200/ce_gmap.py and
graphs.install_ce_gmap_features): the oracle against the reference's own GraphMap and _nav_gmap_variable
(tests/golden/small_ce_gmap.pt) bit for bit, the install's handles against the rows the reference classes gave it, the
merge order the handles record, and install routing."""
import hashlib
import inspect
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import ce_gmap_cases as C  # noqa: E402
from bevbert_b200 import ce_gmap, graphs  # noqa: E402
from oracle import ce_gmap_ref as R  # noqa: E402


class Labels(tuple):
    """an embedding that is the tuple of its (step, env, candidate) labels: `+` concatenates, `/ n` keeps it"""

    def __add__(self, other):
        return Labels(tuple(self) + tuple(other))

    def __truediv__(self, n):
        return self


def drive(gmaps, trainer, seed, mem=None, steps=8):
    """one seeded episode of update_graph calls at B = len(gmaps); a ghost is consumed every third step"""
    rng = np.random.default_rng(seed)
    pos = [rng.uniform(-50, 50, 3) for _ in gmaps]
    for s in range(steps):
        if mem is not None:
            mem.steps.append(None)
        for i, g in enumerate(gmaps):
            n = int(rng.integers(0, 6)) if s != 2 else 0
            cand_pos = C.positions(rng, g, pos[i], n)
            cur = str(len(g.node_pos))
            g.update_graph(None, s + 1, cur, pos[i], Labels([("n", s, i)]), ["%s_%d" % (cur, k) for k in range(n)],
                           cand_pos, [Labels([(s, i, k)]) for k in range(n)], None)
            if s % 3 == 2 and g.ghost_pos:
                g.delete_ghost(next(iter(g.ghost_pos)))
            pos[i] = pos[i] + rng.uniform(-3, 3, 3)


@pytest.mark.parametrize("merge_ghost", [True, False])
def test_handles_record_merge_order(merge_ghost):
    trainer = type("Trainer", (), {})()
    ref = [R.GraphMap(False, 0.5, merge_ghost, 0) for _ in range(4)]
    drive(ref, trainer, 5)
    trainer.gmaps = [R.GraphMap(False, 0.5, merge_ghost, 0) for _ in range(4)]
    mem = ce_gmap.Memory()
    for g in trainer.gmaps:
        ce_gmap.attach(trainer, g, mem)
    drive(trainer.gmaps, trainer, 5, mem)
    merged = 0
    for a, b in zip(ref, trainer.gmaps):
        assert list(a.node_pos) == list(b.node_pos) and list(a.ghost_pos) == list(b.ghost_pos)
        for vp, h in b.node_embeds.items():
            assert [("n", h.s, h.i)] == list(a.node_embeds[vp])
        for vp, (h, n) in b.ghost_embeds.items():
            assert h.terms == tuple(a.ghost_embeds[vp][0]) and n == a.ghost_embeds[vp][1] == len(h.terms)
            merged += n > 1
    assert merged > 0 if merge_ghost else merged == 0


def test_install_routing():
    trainer = C.Trainer(3, "cpu")
    net = trainer.policy.net
    own = trainer._nav_gmap_variable
    graphs.install_ce_gmap_features(trainer)
    assert trainer._nav_gmap_variable is not own
    # other calls of the network pass through untouched and record nothing
    trainer.gmaps = [R.GraphMap(False, 0.5, True, 0)]
    x = torch.zeros(1, 2, C.H)
    out = net(mode="navigation", gmap_img_fts=x, gmap_masks=torch.ones(1, 2, dtype=torch.bool))
    assert out["fused_logits"].shape == (1, 2)
    assert ce_gmap.episode(trainer.gmaps) is None
    # a panorama call attaches the fresh GraphMaps; the CPU outputs are rejected by the memory
    inputs, _ = C.step_inputs(np.random.default_rng(0), 1, "cpu")
    with pytest.raises(TypeError):
        net(mode="panorama", **inputs)
    mem = ce_gmap.episode(trainer.gmaps)
    assert isinstance(mem, ce_gmap.Memory) and mem.steps == []
    # get_node_embeds answers a placeholder, and hands its handle over, while the trainer's own method runs
    g = trainer.gmaps[0]
    g.node_pos["0"], g.node_embeds["0"] = np.zeros(3), ce_gmap.Node(mem, 0, 0)
    out, rows = ce_gmap.trainer_method(lambda: g.get_node_embeds("0"), trainer.gmaps)
    assert out.numel() == 0 and rows == [[g.node_embeds["0"]]] and mem.collect is None
    # GraphMaps of two episodes in one list are refused
    trainer.gmaps.append(R.GraphMap(False, 0.5, True, 0))
    with pytest.raises(RuntimeError):
        ce_gmap.episode(trainer.gmaps)
    with pytest.raises(ValueError):
        ce_gmap.Cands(mem, ((0, 0, 0), (0, 0, 1))) / 3


GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "small_ce_gmap.pt"), weights_only=False)


@pytest.mark.parametrize("ci", range(len(C.GOLDEN_CASES)))
def test_oracle_matches_reference_golden(ci):
    gold = GOLD["cases"][ci]
    assert gold["case"] == C.GOLDEN_CASES[ci]
    t = C.Trainer(3, "cpu")
    steps = C.golden_episode(gold["case"], R.GraphMap, t, t._nav_gmap_variable)
    assert len(steps) == len(gold["steps"])
    for s, ((out, _, dg), g) in enumerate(zip(steps, gold["steps"])):
        assert dg == g["input_digests"], s
        f = out["gmap_img_fts"]
        assert f.dtype == torch.float32 and tuple(f.shape) == g["fts_shape"], s
        assert hashlib.sha256(f.contiguous().numpy().tobytes()).hexdigest() == g["fts_digest"], s
        assert out["gmap_vp_ids"] == g["gmap_vp_ids"] and out["no_vp_left"] == g["no_vp_left"], s


@pytest.mark.parametrize("ci", range(len(C.GOLDEN_CASES)))
def test_install_rows_match_reference_golden(ci):
    """the handles the install collects over the oracle GraphMap and trainer stand-in are those it collected over the
    reference's own GraphMap and _nav_gmap_variable"""
    gold = GOLD["cases"][ci]
    t = C.Trainer(3, "cpu")
    steps = C.golden_episode(gold["case"], R.GraphMap, t, t._nav_gmap_variable, handles=True)
    for s, ((out, rows, _), g) in enumerate(zip(steps, gold["steps"])):
        assert rows == g["rows"] and out["gmap_vp_ids"] == g["gmap_vp_ids"], s
    assert any(len(r) > 1 for g in gold["steps"] for row in g["rows"] for r in row if r[0] != "n") == \
        gold["case"]["merge_ghost"]


def test_install_keeps_the_network_signature():
    """install_ce_waypoint_step binds the network's forward signature, so it may be installed after this install"""
    trainer = C.Trainer(3, "cpu")
    before = inspect.signature(trainer.policy.net.forward)
    graphs.install_ce_gmap_features(trainer)
    assert inspect.signature(trainer.policy.net.forward) == before
