"""The VLN-CE pre-training model (model/ce_pretrain.py) on CPU: its fp32 oracle (oracle/ce_ref.py) against the golden
outputs of the unmodified CE reference, the reference's state_dict surface, the host logic with the kernels emulated,
the BEV known-answer points at 11 x 11 / 1 m, and a rehearsal of the bb_add_rows3 checkers of
tests/test_ce_add_rows3_gpu.py against planted faults."""
import os
import sys

import pytest
import torch

import ce_cases as C
from bevbert_b200 import blocks as Bk
from bevbert_b200 import synth
from bevbert_b200.model.ce_pretrain import GlocalTextPathCMTPreTraining
from helpers import grad_report
from oracle import bevbert_ref as R
from oracle import ce_ref as CR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden():
    sys.path.insert(0, GOLD)
    import make_ce_golden
    return make_ce_golden, torch.load(os.path.join(GOLD, "small_ce.pt"), weights_only=False)


@pytest.fixture
def ce_emu(emu, monkeypatch):
    import bevbert_b200.kernels as K
    monkeypatch.setattr(K, "add_rows", C.emu_add_rows(emu.add_rows))
    return emu


def test_oracle_reproduces_ce_reference():
    mk, gold = _golden()
    cfg, scfg = mk.case()
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=gold["weight_seed"])
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    ocfg = CR.OracleConfig(cfg)
    for task, g in gold["tasks"].items():
        b = synth.make_batch(scfg, seed=gold["batch_seed"], task=task)
        for v in sd.values():
            v.grad = None
        loss = CR.forward(sd, synth.clone_batch(b), task, ocfg)
        loss.mean().backward()
        assert torch.allclose(loss, g["loss"], rtol=1e-5, atol=1e-6), task
        logits = CR.forward({k: v.detach() for k, v in sd.items()}, synth.clone_batch(b), task, ocfg, compute_loss=False)
        logits = logits if isinstance(logits, tuple) else (logits,)
        for a, r in zip(logits[:3], g["logits"]):
            fin = torch.isfinite(r)
            assert torch.equal(torch.isfinite(a), fin)
            assert torch.allclose(a[fin], r[fin], rtol=1e-4, atol=1e-5)
        top = max(g["grad_norms"].values())
        got = {n for n, v in sd.items() if v.grad is not None and n != "mlm_head.predictions.decoder.weight"}
        assert got == set(g["grad_norms"]), got ^ set(g["grad_norms"])
        for n, gn in g["grad_norms"].items():
            tol = 1e-3 * max(gn, 1e-4 * top)
            assert abs(float(sd[n].grad.norm()) - gn) <= tol, (task, n)
            # direction, not only norm: projections on the golden's seeded directions
            proj = mk.grad_projections(n, sd[n].grad)
            assert float((proj - g["grad_proj"][n]).abs().max()) <= tol, (task, n)
        for n, gr in g["grads"].items():
            atol = max(1e-4 * float(gr.abs().max()), 1e-3 * 1e-4 * top) + 1e-9
            assert torch.allclose(sd[n].grad, gr, rtol=1e-3, atol=atol), (task, n)


def test_state_dict_surface_equals_reference():
    """keys, shapes AND order: the reference's build_optimizer groups named_parameters() by position and
    optimizer.load_state_dict restores Adam state by position, so a checkpoint's optimizer state only fits a model whose
    parameters come in the reference's order"""
    mk, gold = _golden()
    cfg, _ = mk.case()
    model = GlocalTextPathCMTPreTraining(cfg)
    assert [(k, tuple(v.shape)) for k, v in model.state_dict().items()] == list(gold["shapes"].items())
    assert [n for n, _ in model.named_parameters()] == gold["param_order"]
    img = "bert.img_embeddings."
    assert gold["shapes"][img + "loc_linear.weight"] == (768, 4)
    assert gold["shapes"][img + "nav_type_embedding.weight"] == (2, 768)
    assert gold["shapes"][img + "dep_linear.weight"] == (768, 128) and img + "dep_layer_norm.weight" in gold["shapes"]
    assert not any(k.startswith("local_sem_head") for k in gold["shapes"]) and "sap_fuse_linear.net.0.weight" in gold["shapes"]
    assert model.bert.bev_dim == 11


def test_from_pretrained_accepts_partial_and_superset_state_dicts():
    mk, _ = _golden()
    cfg, _ = mk.case()
    src = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=5).state_dict()
    part = {k: v for k, v in src.items() if k.startswith("bert.img_embeddings.")}
    part["bert.some_other_head.weight"] = torch.zeros(3)                      # superset key: ignored
    part["bert.img_embeddings.loc_linear.weight"] = torch.zeros(768, 7)        # the discrete shape: ignored
    m = GlocalTextPathCMTPreTraining.from_pretrained(None, config=cfg, state_dict=part)
    sd = m.state_dict()
    assert torch.equal(sd["bert.img_embeddings.dep_linear.weight"], src["bert.img_embeddings.dep_linear.weight"])
    assert not torch.equal(sd["bert.img_embeddings.loc_linear.weight"], src["bert.img_embeddings.loc_linear.weight"])
    assert m.mlm_head.predictions.decoder.weight is m.bert.embeddings.word_embeddings.weight


@pytest.mark.parametrize("task", ["mrc", "og", "valid_sap_og", "sem", "masksem", "bogus"])
def test_unrunnable_tasks_raise_value_error(task):
    mk, _ = _golden()
    cfg, scfg = mk.case()
    model = GlocalTextPathCMTPreTraining(cfg)
    b = synth.make_batch(scfg, seed=1, task="sap")
    with pytest.raises(ValueError, match=task if task != "masksem" else "sem"):
        model(synth.clone_batch(b), task)
    with pytest.raises(ValueError):
        CR.forward({}, synth.clone_batch(b), task, CR.OracleConfig(cfg))


def _host_run(task, cfg, scfg, seed=7, prepare=None):
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).train()
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    b = synth.make_batch(scfg, seed=seed, task=task)
    out = model((prepare or synth.clone_batch)(b), task, compute_loss=True)
    out.mean().backward()
    ref = CR.forward(sd, synth.clone_batch(b), task, CR.OracleConfig(cfg))
    ref.mean().backward()
    assert out.shape == ref.shape
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-5), float((out - ref).abs().max())
    worst, name = grad_report({n: p.grad for n, p in model.named_parameters()},
                              {n: sd[n].grad for n, _ in model.named_parameters()})
    assert worst < 1e-3, (worst, name)
    return out, {n: p.grad for n, p in model.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("task", ["mlm", "sap"])
def test_host_logic_matches_oracle_and_prepare_batch_changes_nothing(ce_emu, task):
    from bevbert_b200.model.ops import prepare_batch
    mk, _ = _golden()
    cfg, scfg = mk.case()
    scfg.ragged_txt = True
    out, grads = _host_run(task, cfg, scfg, seed=13)
    out2, grads2 = _host_run(task, cfg, scfg, seed=13, prepare=lambda b: prepare_batch(synth.clone_batch(b)))
    assert torch.equal(out, out2)
    for n, g in grads.items():
        assert torch.equal(g, grads2[n]), n


def test_prepare_batch_ships_depth_features_in_the_wire_format():
    from bevbert_b200.model.ops import prepare_batch
    mk, _ = _golden()
    _, scfg = mk.case()
    b = synth.make_batch(scfg, seed=3, task="sap")
    assert "sems" not in b and b["traj_loc_fts"].shape[-1] == 4 and b["traj_view_img_fts"].shape[-1] == 512
    assert b["traj_view_dep_fts"].shape[:2] == b["traj_view_img_fts"].shape[:2] and b["traj_view_dep_fts"].shape[-1] == 128
    assert set(b["traj_nav_types"].unique().tolist()) <= {0, 1} and int(b["bev_cand_idxs"].max()) < 121
    w = prepare_batch(synth.clone_batch(b), wire_dtype=torch.bfloat16)
    for k in ("rgbs", "traj_view_img_fts", "traj_view_dep_fts"):
        assert w[k].dtype == torch.bfloat16 and torch.equal(w[k], b[k].to(torch.bfloat16)), k
    # every tensor but the depth features and the 4 location columns is the R2R batch of the same seed
    r2r = synth.make_batch(synth.SynthConfig(**dict(vars(scfg), depth_feat_size=0)), seed=3, task="sap")
    for k, v in b.items():
        if torch.is_tensor(v) and k not in ("traj_view_dep_fts", "traj_loc_fts"):
            assert torch.equal(v, r2r[k]), k
    assert torch.equal(b["traj_loc_fts"], r2r["traj_loc_fts"][..., :4])


def test_lift_known_answers_at_11_cells_1m():
    pts, nod, want = C.lift_kat_points()
    assert torch.equal(R.cell_index(pts, nod, C.D_CE, C.RES_CE)[0], want)
    b = synth.make_batch(synth.ce_synth_config(batch_size=2), seed=5, task="sap")
    out = CR.lift_splat(dict(b))
    assert out["bev_fts"].shape == (2, 121, 768) and out["bev_pos_fts"].shape == (2, 121, 10)
    assert out["bev_masks"].all() and "bev_sems" not in out


@pytest.mark.parametrize("case", C.CASES[:6])
def test_add_rows3_checkers_pass_emulation_and_reject_planted_faults(case):
    act = torch.bfloat16
    emu = C.emu_add_rows(lambda a, *r: a.to(act))

    def run(fault=None):
        ops = C.make_case(case, act, seed=1)
        rows, H = ops["a"].shape
        emu(ops["a"], ops["b"], ops["table"], ops["idx"], ops["vec"], c=ops["c"], out=ops["out"])
        if fault == "ulp":
            v = ops["out"][rows // 2, H - 1:H]
            v.copy_((v.view(torch.int16) + 1).view(act))                      # one bf16 ulp
        elif fault == "pad_read":
            ops["out"][rows - 1, H - 1] += ops["a_buf"][rows - 1, -1] if ops["a_buf"].shape[1] > H else \
                ops["a_buf"][rows, 0]
        elif fault == "write_past_end":
            ops["out_buf"][rows + 1, 0] = 0
        elif fault == "drop_c":
            ops["out"].copy_((ops["out"].float() - ops["c"].float()).to(act))
        return ops

    C.check_forward(run(), act, "clean")
    for fault in ("ulp", "pad_read", "write_past_end", "drop_c"):
        with pytest.raises(AssertionError):
            C.check_forward(run(fault), act, fault)


def test_add_rows3_backward_checker(emu, monkeypatch):
    import bevbert_b200.kernels as K
    monkeypatch.setattr(K, "add_rows", C.emu_add_rows(emu.add_rows))
    ops = C.make_case(C.CASES[2], torch.float32, seed=2)
    vsrc = torch.stack([torch.randn(ops["a"].shape[1]), ops["vec"]])
    impl, st = Bk.AddRows3Impl(vec_row=1), {}
    impl.fwd(st, [ops["a"], ops["b"], ops["c"], ops["idx"]], [ops["table"], vsrc])
    g = torch.randn(ops["a"].shape).to(emu.ACT)
    gin, gp = impl.bwd(st, [g], [ops["table"], vsrc])
    C.check_backward(g, (gin, gp), ops, "emulated")
    with pytest.raises(AssertionError):
        C.check_backward(g, ([gin[0], gin[1], None, None], gp), ops, "dc dropped")
    with pytest.raises(AssertionError):
        C.check_backward(g, (gin, (gp[0] * 1.001, gp[1])), ops, "dtable off")


def test_encoder_forward_takes_return_gmap_embeds(ce_emu):
    """GlocalTextPathCMT.forward(..., return_gmap_embeds=False) -> (None, bev_embeds), as CE vilmodel.py:726-774"""
    from collections import defaultdict
    mk, _ = _golden()
    cfg, scfg = mk.case()
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).eval()
    b = model.lift_splat(defaultdict(lambda: None, synth.make_batch(scfg, seed=5, task="sap")))
    model.rt.begin(False, tag="sap")
    model.drop_feats(b)
    args = [b[k] for k in model._BERT_KEYS]
    with torch.no_grad():
        g0, bev0 = model.bert(*args, return_gmap_embeds=False)
        g1, bev1 = model.bert(*args)
    assert g0 is None and g1 is not None and g1.shape[:2] == b["gmap_step_ids"].shape
    assert bev0.shape == (scfg.batch_size, 121, cfg.hidden_size) and torch.equal(bev0, bev1)


def test_add_rows_takes_out_only_with_the_third_operand():
    import bevbert_b200.kernels as K
    with pytest.raises(ValueError, match="out"):
        K.add_rows(torch.zeros(2, 8), out=torch.zeros(2, 8))
