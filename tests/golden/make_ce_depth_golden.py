"""Generates tests/golden/small_ce_depth.pt by running the UNMODIFIED depth encoder wrapper of the VLN-CE policy
(bevbert_ce/vlnce_baselines/models/encoders/resnet_encoders.py::VlnResnetDepthEncoder), from the reference checkout
located by oracle/ref_shim.py (env BEVBERT_REFERENCE):

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_ce_depth_golden.py

resnet_encoders.py imports gym.spaces, habitat.logger, vlnce_baselines.models.encoders.clip and habitat-lab's
`habitat_baselines.rl.ddppo.policy.{resnet, resnet_policy}`; those are stub modules here, the last two backed by
bevbert_b200/model/depth_resnet.py (habitat-lab's source is not available, so the backbone is pinned to the restated
layout, not to habitat-lab).  This pins the wrapper: its strict load of a DD-PPO checkpoint through the
`k.split(".")[2:]` remap (synth.ddppo_checkpoint(SEED), saved with torch.save and loaded by the wrapper's own
torch.load), its `depth_features` passthrough and its `spatial_output=True` shape.

Stored (data only): the wrapper's loaded visual_encoder key -> shape map in order; outputs at N = 2 in fp32 and fp64;
the passthrough check; the spatial output shape."""
import importlib
import os
import sys
import tempfile
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT]

from bevbert_b200 import synth  # noqa: E402
from bevbert_b200.model import depth_resnet as D  # noqa: E402
from oracle import ref_shim  # noqa: E402

SEED, DEPTH_SEED, N = 41, 42, 2
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "small_ce_depth.pt")


def _pkg(name, path=None):
    m = types.ModuleType(name)
    if path is not None:
        m.__path__ = [path]
    sys.modules[name] = m
    return m


def load_reference():
    base = os.path.join(ref_shim.REF_ROOT, "bevbert_ce", "vlnce_baselines")
    if not os.path.isdir(base):
        raise RuntimeError("CE reference tree not found under %s" % ref_shim.REF_ROOT)
    sys.dont_write_bytecode = True
    gym = _pkg("gym")
    gym.spaces = _pkg("gym.spaces")
    gym.spaces.Dict = D.Spaces
    gym.spaces.Box = lambda low, high, shape, dtype=None: D.Box(shape)
    _pkg("habitat").logger = None
    _pkg("habitat_baselines")
    _pkg("habitat_baselines.rl")
    _pkg("habitat_baselines.rl.ddppo")
    pol = _pkg("habitat_baselines.rl.ddppo.policy")
    pol.resnet = _pkg("habitat_baselines.rl.ddppo.policy.resnet")
    pol.resnet.resnet50 = D.resnet50
    pol.resnet_policy = _pkg("habitat_baselines.rl.ddppo.policy.resnet_policy")
    pol.resnet_policy.ResNetEncoder = D.ResNetEncoder
    _pkg("vlnce_baselines", base)
    _pkg("vlnce_baselines.models", os.path.join(base, "models"))
    enc = _pkg("vlnce_baselines.models.encoders", os.path.join(base, "models", "encoders"))
    enc.clip = _pkg("vlnce_baselines.models.encoders.clip")
    return importlib.import_module("vlnce_baselines.models.encoders.resnet_encoders")


def main():
    re = load_reference()
    space = D.Spaces({"depth": D.Box((256, 256, 1))})
    with tempfile.TemporaryDirectory() as d:
        ck = os.path.join(d, "gibson-2plus-resnet50.pth")
        torch.save(synth.ddppo_checkpoint(SEED), ck)
        m = re.VlnResnetDepthEncoder(space, output_size=128, checkpoint=ck, backbone="resnet50",
                                     resnet_baseplanes=32, normalize_visual_inputs=False, trainable=False,
                                     spatial_output=False).eval()
    depth = synth.depth_images(N, DEPTH_SEED)
    with torch.no_grad():
        out32 = m({"depth": depth})
        out64 = m.double()({"depth": depth.double()})
        m.float()
        feats = torch.randn(N, 128, 4, 4, generator=torch.Generator().manual_seed(3))
        passthrough = bool(torch.equal(m({"depth_features": feats}), feats))
        sp = re.VlnResnetDepthEncoder(space, spatial_output=True).eval()
        spatial_shape = tuple(sp({"depth": depth}).shape)
    torch.save({"seed": SEED, "depth_seed": DEPTH_SEED, "n": N,
                "keys": [(k, tuple(v.shape)) for k, v in m.visual_encoder.state_dict().items()],
                "out_fp32": out32, "out_fp64": out64, "passthrough": passthrough,
                "spatial_shape": spatial_shape,
                "params_requires_grad": any(p.requires_grad for p in m.visual_encoder.parameters())}, OUT)
    print("wrote %s: %d keys, out %s, spatial %s" % (OUT, len(m.visual_encoder.state_dict()), tuple(out32.shape),
                                                     spatial_shape))


if __name__ == "__main__":
    main()
