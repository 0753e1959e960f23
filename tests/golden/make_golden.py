"""Generates tests/golden/*.pt by running the UNMODIFIED reference (located by oracle/ref_shim.py, env
BEVBERT_REFERENCE) on seeded weights and synthetic batches.  Needs a checkout of the reference:

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_golden.py

reference_pins.pt holds what tests/test_oracle_vs_reference.py, tests/test_optim_cpu.py and tests/test_nav_api_cpu.py
compare the restatements with (reference outputs on the batches those tests build; large tensors as a seeded sample
of rows plus float64 sums), so the suite needs no reference checkout.

Weights (synth.det_init_) and batches (synth.make_batch) are regenerated bit-identically from their seeds by
the tests, so only reference OUTPUTS are stored: per-item losses, logits, per-parameter gradient norms and a
few full gradients.  The reference has no tests or golden vectors of its own (SURVEY.md 4)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bevbert_b200 import synth  # noqa: E402
from bevbert_b200.model.pretrain_cmt import GlocalTextPathCMTPreTraining  # noqa: E402
from helpers import small_config, small_synth  # noqa: E402
from oracle import ref_shim  # noqa: E402

FULL_GRADS = ["bert.embeddings.LayerNorm.weight", "bert.lang_encoder.layer.0.attention.self.query.bias",
              "bert.local_encoder.encoder.x_layers.0.visual_attention.att.query.bias",
              "bert.global_encoder.sprel_linear.weight", "bert.global_encoder.sprel_linear.bias",
              "bert.img_embeddings.loc_linear.weight", "bert.local_encoder.bev_pos_embeddings.0.weight"]

CASES = {
    "small_r2r": (lambda: small_config(), lambda: small_synth(), ["mlm", "sap", "masksem"]),
    "small_reverie": (lambda: small_config(obj_feat_size=768, obj_prob_size=100, pretrain_tasks=["mlm", "mrc", "sap", "og"]),
                      lambda: small_synth(obj_feat_size=768, obj_max=5, obj_prob_size=100), ["mlm", "mrc", "sap", "og"]),
}


def main():
    out_dir = os.path.dirname(os.path.abspath(__file__))
    for name, (mk_cfg, mk_synth, tasks) in CASES.items():
        cfg, scfg = mk_cfg(), mk_synth()
        ours = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3)
        sd = {k: v.detach().clone() for k, v in ours.state_dict().items()}
        ref = ref_shim.build_reference_model(cfg, sd).train()
        for m in ref.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
            if isinstance(m, torch.nn.MultiheadAttention):
                m.dropout = 0.0
        assert set(ref.state_dict().keys()) == set(sd.keys()), "state_dict key sets differ"
        for k, v in ref.state_dict().items():
            assert v.shape == sd[k].shape, k
        gold = {"state_dict_keys": sorted(sd.keys()), "shapes": {k: tuple(v.shape) for k, v in sd.items()}}
        for task in tasks:
            b = synth.make_batch(scfg, seed=7, task=task)
            ref.zero_grad()
            loss = ref(synth.clone_batch(b), task, compute_loss=True)
            loss.mean().backward()
            with torch.no_grad():
                logits = ref(synth.clone_batch(b), task, compute_loss=False)
            logits = logits if isinstance(logits, tuple) else (logits,)
            grads = {n: p.grad for n, p in ref.named_parameters() if p.grad is not None}
            gold[task] = {
                "loss": loss.detach().clone(),
                "logits": [t.detach().clone() for t in logits[:3]],
                "grad_norms": {n: float(g.norm()) for n, g in grads.items()},
                "grads": {n: grads[n].clone() for n in FULL_GRADS if n in grads},
            }
            print(name, task, "loss mean %.6f" % float(loss.mean()), "n_grads", len(grads))
        torch.save(gold, os.path.join(out_dir, name + ".pt"))


def sample_rows(x, n=16, seed=0):
    """Fixed, seeded sample of n rows of x flattened to 2-D, plus float64 sums of the whole tensor."""
    x2 = x.reshape(-1, x.shape[-1]).detach()
    idx = torch.randperm(x2.shape[0], generator=torch.Generator().manual_seed(seed))[:n].sort().values
    return {"idx": idx, "rows": x2[idx].clone(), "sum": float(x2.double().sum()), "abs_sum": float(x2.double().abs().sum())}


def pins():
    import test_nav_api_cpu as nav_t
    import test_optim_cpu as opt_t
    import test_oracle_vs_reference as ovr
    out = {"restatement": {}, "edge": {}, "bev": [], "adamw": {}, "nav": {}}
    cfg = small_config()
    sd = {k: v.detach().clone() for k, v in synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=5).state_dict().items()}
    ref = ovr._ref_model(cfg, sd)
    for task in ("mlm", "sap", "masksem"):
        b = synth.make_batch(small_synth(ragged_txt=True), seed=21, task=task)
        out["restatement"][task] = ref(synth.clone_batch(b), task, compute_loss=True).detach().clone()
    for case in ("longest_trajectory", "empty_bev"):
        scfg = small_synth(pano_min=21, pano_max=21) if case == "longest_trajectory" else small_synth(depth_zero_frac=1.0)
        for task in ("sap", "mlm"):
            b = synth.make_batch(scfg, seed=23, task=task)
            out["edge"][case + "/" + task] = ref(synth.clone_batch(b), task, compute_loss=True).detach().clone()
    _, pretrain_cmt = ref_shim.load_pretrain_modules(21, 0.5)
    projector, _ = pretrain_cmt.build_projector()
    for seed in (1, 2, 3):
        b = synth.make_batch(synth.SynthConfig(batch_size=4), seed=seed)
        bs = 4
        depths = (b["depths"] * 10).reshape(-1, 1, 14, 14)
        pc, mask = projector.forward(depths, b["T_c2w"].reshape(-1, 4, 4))
        pc = pc.reshape(bs, -1, 3) - b["S_w2c"]
        pc1 = torch.cat([pc, torch.ones(bs, pc.shape[1], 1)], -1) @ b["T_w2c"].squeeze(1).transpose(1, 2)
        bev, ob, sem, sem_mask = projector.project_bev(pc1[:, :, :3], mask.reshape(bs, -1), b["rgbs"].reshape(bs, -1, 768),
                                                       b["sems"].reshape(bs, -1, 40))
        from oracle import bevbert_ref as R
        ref_idx = R.cell_index(pc1[:, :, :3], mask.reshape(bs, -1), 21, 0.5)
        out["bev"].append({"cell_idx": ref_idx.to(torch.int16), "bev": sample_rows(bev.reshape(bs, -1, 768), 64, seed),
                           "sems": sample_rows(sem.reshape(bs, -1, 40), 64, seed), "sem_masks": sem_mask.reshape(bs, -1).clone(),
                           "ob_masks": ob.reshape(bs, -1).clone()})
    a = opt_t._params()
    opt = opt_t._ref_adamw()([{"params": [a[0], a[2], a[3]], "weight_decay": 0.01}, {"params": [a[1]], "weight_decay": 0.0}],
                             lr=3e-3, betas=(0.9, 0.98))
    g = torch.Generator().manual_seed(2)
    norms = []
    for step in range(9):
        grads = [torch.randn(p.shape, generator=g) * (10.0 if step == 4 else 1.0) for p in a]
        for i, p in enumerate(a):
            p.grad = None if i == step % 4 else grads[i].clone()
        norms.append(float(torch.nn.utils.clip_grad_norm_(a, 5.0)))
        opt.step()
    out["adamw"] = {"clip_norms": norms, "params": [p.detach().clone() for p in a]}
    ncfg = nav_t.nav_config()
    nav_mod = ref_shim.load_nav_module()
    nsd = {k: v.detach().clone() for k, v in synth.det_init_(nav_t.GlocalTextPathNavCMT(ncfg), seed=4).state_dict().items()}
    nref = nav_mod.GlocalTextPathNavCMT(ncfg)
    nref.load_state_dict(nsd)
    nref.eval()
    lang, pano, nav = nav_t.nav_batches()
    with torch.no_grad():
        t = nref("language", lang)
        pe, pm = nref("panorama", pano)
        nav["txt_embeds"] = t
        want = nref("navigation", nav)
    out["nav"] = {"state_dict_keys": sorted(nref.state_dict().keys()), "language": sample_rows(t, 24, 1), "panorama": sample_rows(pe, 24, 2), "panorama_masks": pm.clone(),
                  "navigation": {k: want[k].detach().clone() for k in ("global_logits", "local_logits", "fused_logits")},
                  "gmap_embeds": sample_rows(want["gmap_embeds"], 16, 3)}
    torch.save(out, os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_pins.pt"))


if __name__ == "__main__":
    main()
    pins()
