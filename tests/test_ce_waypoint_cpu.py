"""CPU checks of the VLN-CE waypoint predictor and its heatmap NMS (model/waypoint.py): the oracle
(oracle/ce_waypoint_ref.py) against the unmodified reference (tests/golden/small_ce_waypoint.pt), the state_dict
surface, the neighbour bias, and the host logic of the NMS wrapper and of the predictor install."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevbert_b200 import graphs, synth  # noqa: E402
from bevbert_b200.model import waypoint as WP  # noqa: E402
from oracle import ce_waypoint_ref as R  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "small_ce_waypoint.pt")
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_ce_waypoint_golden as MG  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.mark.parametrize("B", MG.BATCHES)
def test_oracle_predictor_matches_reference_golden(golden, B):
    sd = synth.waypoint_state(golden["seed"])
    got = MG.summarize(R.forward(sd, MG.depth_feats(B, golden["feat_seed"]), torch.float64))
    for k, ref in golden["logits_B%d" % B].items():
        err = float((got[k] - ref).abs().max() / ref.abs().max())
        assert err < 1e-5, (k, err)       # reference: fp32 on the CPU; oracle: fp64


def test_oracle_nms_bit_identical_on_every_golden_case(golden):
    assert len(golden["nms"]) == 19
    for name, c in golden["nms"].items():
        got = R.nms(c["pred"], c["k"], c["sigma"])
        assert torch.equal(got.view(torch.int32), c["out"].view(torch.int32)), name
        dev = R.nms_device(c["pred"], c["k"], c["sigma"])   # the timed reference path, on the CPU
        assert torch.equal(dev.view(torch.int32), c["out"].view(torch.int32)), name


def test_oracle_footprint_table(golden):
    fp = R.footprint()
    assert torch.equal(torch.from_numpy(np.packbits(fp.numpy(), axis=-1)), golden["footprint"])
    # a peak at row 10, column 0 suppresses rows 5-15 and columns 0-7 (the circular distance is not symmetric); at
    # column 5 or 11, y_mu = 10 + col / 12 keeps rows 6-15 and every column is within 7
    for col, rows, cols in ((0, range(5, 16), range(0, 8)), (5, range(6, 16), range(12)), (11, range(6, 16), range(12))):
        box = torch.zeros(122, 12, dtype=torch.bool)
        box[list(rows)[0]:list(rows)[-1] + 1, list(cols)[0]:list(cols)[-1] + 1] = True
        assert torch.equal(fp[10 * 12 + col].view(122, 12), box), col


def test_policy_rows_agree_under_reciprocal_division():
    """y_mu = ix / 12 correctly rounded (the reference on the CPU) and ix * fp32(1/12) (torch's CUDA form of a division
    by a scalar) keep the same rows at every centre of the policy's map"""
    ix = torch.arange(122 * 12, dtype=torch.float32)
    exact = ix / 12.0
    recip = ix * torch.tensor(1.0 / 12.0, dtype=torch.float32)
    y = torch.arange(122, dtype=torch.float32).view(1, -1)
    assert torch.equal((y - exact.view(-1, 1)).abs() <= 5.0, (y - recip.view(-1, 1)).abs() <= 5.0)


def test_state_dict_surface(golden):
    m = WP.BinaryDistPredictor_TRM()
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [tuple(x) for x in golden["keys"]]
    assert list(synth.waypoint_state(0).keys()) == list(m.state_dict().keys())
    m.load_state_dict(synth.waypoint_state(3))          # strict
    assert [n for n, _ in m.named_parameters()] == [k for k, _ in golden["keys"]]


def test_neighbour_bias(golden):
    mask = golden["attention_mask"]                     # utils.get_attention_mask(12, 1), (1, 1, 12, 12) int64
    assert torch.equal(WP.neighbour_mask(), mask[0, 0])
    assert torch.equal(R.neighbour_mask(), mask[0, 0])
    runner = WP.WaypointRunner(WP.BinaryDistPredictor_TRM())
    for B in (1, 3):
        ref = ((1.0 - mask.to(torch.float32)) * -10000.0).repeat(B, 1, 1, 1)[:, 0]
        got = runner.bias(B, torch.device("cpu"))
        assert got.dtype == torch.float32 and got.is_contiguous() and torch.equal(got, ref)
        assert runner.bias(B, torch.device("cpu")) is got
        assert torch.equal(R.neighbour_bias(B)[:, 0], ref)


def test_nms_rejections():
    x = torch.zeros(2, 1, 122, 12)
    with pytest.raises(NotImplementedError):
        WP.nms(x, 5, (7.0, 5.0), gaussian=True)
    with pytest.raises(TypeError):
        WP.nms(x.double(), 5, (7.0, 5.0))
    with pytest.raises(TypeError):
        WP.nms(x.half(), 5, (7.0, 5.0))
    with pytest.raises(RuntimeError, match="CUDA"):
        WP.nms(x, 5, (7.0, 5.0))
    assert WP.NMS_MAX_CELLS >= 122 * 12


class _FakeCuda:
    """a CPU tensor that reports is_cuda, to reach the shape checks that come after the device check"""

    def __init__(self, shape):
        self.shape, self.dtype, self.is_cuda = torch.Size(shape), torch.float32, True

    def dim(self):
        return len(self.shape)


@pytest.mark.parametrize("shape", [(2, 122, 12), (2, 2, 122, 12), (1, 1, 91, 91), (1, 1, 8193, 1)])
def test_nms_shape_and_size_rejections(shape):
    with pytest.raises(ValueError):
        WP.nms(_FakeCuda(shape), 5, (7.0, 5.0))


def _policy():
    """the trainer's attributes: a frozen predictor in eval mode, wrapped in DataParallel or not"""
    wp = WP.BinaryDistPredictor_TRM()
    wp.requires_grad_(False).eval()
    return wp


@pytest.mark.parametrize("wrap", [False, True])
def test_install_host_logic(wrap):
    wp = _policy()
    outer = torch.nn.DataParallel(wp) if wrap else wp
    before = {k: v.clone() for k, v in outer.state_dict().items()}
    replay = graphs.install_ce_waypoint_predictor(outer)
    after = outer.state_dict()
    assert list(after) == list(before) and all(torch.equal(after[k], v) for k, v in before.items())
    assert "forward" in wp.__dict__                    # routed on the wrapped module itself
    runner = replay.model
    assert runner.m is wp and replay.s is graphs.CE_WAYPOINT and replay.s.grad_ok
    rgb, dep = torch.zeros(12, 512), torch.zeros(12, 128, 4, 4)
    # training mode raises before anything runs, eval mode follows the module's own switch
    outer.train()
    assert runner.training
    with pytest.raises(RuntimeError, match="eval mode"):
        wp(rgb, dep)
    outer.eval()
    assert not runner.training
    # a parameter that requires grad, with grad enabled, is refused
    wp.vis_classifier[2].bias.requires_grad_(True)
    with pytest.raises(RuntimeError, match="forward only"):
        wp(rgb, dep)
    wp.vis_classifier[2].bias.requires_grad_(False)
    # B comes from rgb_feats.size(0) // 12 and depth_feats must hold its 12 B views
    for r, d in ((torch.zeros(11, 512), dep), (torch.zeros(24, 512), dep), (rgb, torch.zeros(12, 64, 4, 4))):
        with pytest.raises(ValueError):
            wp(r, d)
    with pytest.raises(TypeError):
        wp(rgb, dep.double())
    assert runner.check_inputs(torch.zeros(25, 512), torch.zeros(24, 2048)).shape == (24, 2048)
    # weight changes are seen through storage and version
    assert runner.changed() and not runner.changed()
    wp.load_state_dict(synth.waypoint_state(1))
    assert runner.changed() and not runner.changed()


def test_geometry_is_validated():
    with pytest.raises(ValueError):
        WP.WaypointRunner(WP.BinaryDistPredictor_TRM(hidden_dim=512))
    with pytest.raises(ValueError):
        WP.WaypointRunner(WP.BinaryDistPredictor_TRM(n_classes=6))


def test_replay_key_is_the_exact_view_count():
    def key(n, dt=torch.float32):
        return graphs._bucket(graphs.CE_WAYPOINT_DIMS, "waypoint", {"depth_feats": torch.zeros(n, 128, 4, 4, dtype=dt)})
    assert key(96) != key(84) != key(12)
    assert key(12) == key(12) and key(12) != key(12, torch.float16)
    assert key(12)[2] == ((12, 128, 4, 4), torch.float32)
