"""Generates tests/golden/small_ce_clip.pt by running the UNMODIFIED CLIP image tower of the VLN-CE policy
(bevbert_ce/vlnce_baselines/models/encoders/clip/model.py::VisionTransformer of the reference checkout located by
oracle/ref_shim.py, env BEVBERT_REFERENCE) behind torchvision's ConvertImageDtype(float) + Normalize, composed as
CLIPEncoderB16.forward composes them (encoders/resnet_encoders.py:305-314):

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_ce_clip_golden.py

`clip/__init__.py` imports the model downloader, so model.py is imported through stub parent packages whose
`__path__` points at the reference directories and whose own `__init__` never runs.  Weights are
bevbert_b200.synth.clip_visual_state(SEED) (ViT-B/16 shapes, fp16-rounded where convert_weights stores fp16), run in
fp32 on the CPU as clip.load does there; the input is synth.clip_images(3, IMG_SEED), full 224 x 224 uint8.

Stored (data only): the state_dict key -> shape map; of rgb_vector (3 x 512) the first 16 channels and the row norms;
of rgb_grid (3 x 196 x 768) the first 16 channels of tokens 0, 97 and 195, every token's row norm, and the projection
of each image's grid on PROBES seeded directions; of the preprocessed images a corner and the per-image sums."""
import importlib
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT]

from bevbert_b200 import synth  # noqa: E402
from oracle import ref_shim  # noqa: E402

SEED, IMG_SEED, PROBES = 11, 12, 4
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "small_ce_clip.pt")


def probes(shape):
    """the seeded directions the grid is projected on, (PROBES, *shape)"""
    return synth.det_uniform((PROBES,) + tuple(shape), 77, 1, -1.0, 1.0).double()


def summarize(vec, grid):
    vec, grid = vec.double(), grid.double()
    return {"vec_first": vec[:, :16], "vec_norm": vec.norm(dim=-1), "grid_first": grid[:, [0, 97, 195], :16],
            "grid_norm": grid.norm(dim=-1), "grid_proj": torch.einsum("ntd,ptd->np", grid, probes(grid.shape[1:]))}


def _pkg(name, path):
    m = types.ModuleType(name)
    m.__path__ = [path]
    sys.modules[name] = m
    return m


def load_clip_model():
    base = os.path.join(ref_shim.REF_ROOT, "bevbert_ce", "vlnce_baselines")
    if not os.path.isdir(base):
        raise RuntimeError("CE reference tree not found under %s" % ref_shim.REF_ROOT)
    sys.dont_write_bytecode = True
    _pkg("vlnce_baselines", base)
    _pkg("vlnce_baselines.models", os.path.join(base, "models"))
    _pkg("vlnce_baselines.models.encoders", os.path.join(base, "models", "encoders"))
    _pkg("vlnce_baselines.models.encoders.clip", os.path.join(base, "models", "encoders", "clip"))
    m = importlib.import_module("vlnce_baselines.models.encoders.clip.model")
    assert m.__file__.startswith(base), m.__file__
    return m


def main():
    from torchvision import transforms
    model = load_clip_model()
    sd = synth.clip_visual_state(SEED)
    vit = model.VisionTransformer(**synth.CLIP_B16)
    vit.load_state_dict(sd)
    vit.requires_grad_(False).eval()
    rgb = synth.clip_images(3, IMG_SEED)
    tf = torch.nn.Sequential(transforms.ConvertImageDtype(torch.float),
                             transforms.Normalize([0.48145466, 0.4578275, 0.40821073],
                                                  [0.26862954, 0.26130258, 0.27577711]))
    x = tf(rgb.permute(0, 3, 1, 2))
    with torch.no_grad():
        vec, grid = vit(x.contiguous())
    out = summarize(vec.float(), grid.float())
    out.update(keys=[(k, tuple(v.shape)) for k, v in vit.state_dict().items()], pre_corner=x[:, :, :4, :4].clone(),
               pre_sum=x.double().sum(dim=(1, 2, 3)), seed=SEED, img_seed=IMG_SEED)
    torch.save(out, OUT)
    print("wrote %s" % OUT)


if __name__ == "__main__":
    main()
