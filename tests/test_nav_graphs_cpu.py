"""Shape buckets of the graphed per-step API (bevbert_b200.graphs.GraphedNavigation) on CPU with emulated kernels:
the bucket keys, and the model on zero-padded inputs, sliced back, against the model on the caller's inputs."""
import pytest
import torch

from bevbert_b200 import synth
from bevbert_b200.graphs import nav_bucket, nav_forward_padded, nav_pad, nav_slice
from bevbert_b200.model.nav_vilmodel import GlocalTextPathNavCMT
from test_nav_api_cpu import nav_batches, nav_config


def _close(a, b, what):
    fa, fb = torch.isfinite(a), torch.isfinite(b)
    assert a.shape == b.shape and torch.equal(fa, fb), what
    assert torch.allclose(a[fa], b[fb], rtol=1e-5, atol=1e-5), (what, float((a[fa] - b[fb]).abs().max()))


def test_bucket_keys_round_every_variable_length_to_eight():
    lang, pano, nav = nav_batches(B=3, G=9, K=4)
    nav["txt_embeds"] = torch.zeros(3, 30, 768)
    k = dict(zip(["txt_embeds", "txt_masks", "gmap_img_embeds", "gmap_step_ids", "gmap_pos_fts", "gmap_masks",
                  "gmap_pair_dists", "gmap_visited_masks", "bev_fts", "bev_pos_fts", "bev_masks", "bev_nav_masks",
                  "bev_cand_idxs", "obj_embeds", "obj_masks"], nav_bucket("navigation", nav)[2:]))
    assert k["txt_embeds"] == ((3, 32, 768), torch.float32) and k["txt_masks"] == ((3, 32), torch.bool)
    assert k["gmap_pair_dists"][0] == (3, 16, 16) and k["gmap_masks"][0] == (3, 16)
    assert k["bev_fts"][0] == (3, 121, 768) and k["bev_cand_idxs"][0] == (3, 8)
    assert k["obj_embeds"] is None
    assert nav_bucket("language", lang)[2] == ((3, 32), lang["txt_ids"].dtype)
    # both sides of a bucket edge
    assert nav_bucket("navigation", nav_batches(B=3, G=8)[2]) != nav_bucket("navigation", nav_batches(B=3, G=9)[2])
    assert nav_bucket("navigation", nav_batches(B=3, G=9)[2]) == nav_bucket("navigation", nav_batches(B=3, G=16)[2])
    _, p5, _ = nav_batches(obj=5)
    kp = nav_bucket("panorama", p5)
    assert kp[2][0] == (3, 40, 768) and kp[3][0] == (3, 8, 768) and kp[4][0] == (3, 48, 7)
    assert nav_bucket("panorama", pano)[3] is None


@pytest.mark.parametrize("obj", [0, 5])
@pytest.mark.parametrize("G,K", [(7, 4), (9, 3)])
def test_padded_eager_equals_unpadded_eager(emu, obj, G, K):
    cfg = nav_config(**(dict(obj_feat_size=768) if obj else {}))
    model = synth.det_init_(GlocalTextPathNavCMT(cfg), seed=4).eval()
    lang, pano, nav = nav_batches(G=G, K=K, obj=obj)
    with torch.no_grad():
        t = model("language", lang)
        _close(nav_slice("language", nav_forward_padded(model, "language", nav_pad("language", lang, "cpu")), lang), t,
               "language")
        pe, pm = model("panorama", pano)
        qe, qm = nav_slice("panorama", nav_forward_padded(model, "panorama", nav_pad("panorama", pano, "cpu")), pano)
        assert torch.equal(qm, pm)
        _close(qe, pe, "panorama")
        nav["txt_embeds"] = t
        if obj:
            nav["obj_embeds"] = pe[:, 36:36 + obj]
            nav["obj_masks"] = pm[:, 36:36 + obj]
        ref = model("navigation", nav)
        got = nav_slice("navigation", nav_forward_padded(model, "navigation", nav_pad("navigation", nav, "cpu"),
                                                         (nav["gmap_vpids"], nav["bev_cand_vpids"])), nav)
    for k in ("gmap_embeds", "global_logits", "local_logits", "fused_logits") + (("obj_logits",) if obj else ()):
        _close(got[k], ref[k], k)
    assert (got["obj_logits"] is None) == (not obj)


def test_wrapped_forward_runs_grad_enabled_calls_on_the_model(emu):
    """`inner.forward = GraphedNavigation(inner)` (the agent-side wrapping): calls with gradients run the model itself."""
    from bevbert_b200.graphs import GraphedNavigation
    model = synth.det_init_(GlocalTextPathNavCMT(nav_config()), seed=4).train()
    lang, _, _ = nav_batches()
    ref = model("language", lang)
    model.forward = GraphedNavigation(model)
    got = model("language", lang)
    assert got.requires_grad and torch.equal(got, ref)
    assert not model.forward.entries
