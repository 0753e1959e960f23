"""Deterministic mode: under torch.use_deterministic_algorithms(True) every kernel of the library gives bit-identical
results for bit-identical inputs, whatever else runs on the GPU, and stays as accurate as the default atomics.

Each test runs its case in a fresh interpreter with CUBLAS_WORKSPACE_CONFIG set, because cuBLAS reads that variable
when it initialises.  `python tests/test_deterministic_gpu.py <case>` runs one case directly."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = ["gemm_split_k", "row_reductions", "scatter_exact", "graph_bias", "mt_sumsq", "train_steps", "graph_replay",
         "oracle_bars", "nav_step", "fused_scores_raises"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_deterministic(case):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] +
                                        ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    if case == "fused_scores_raises":
        env.update(BB_FLASH="0", BB_FUSED_SCORES_MAX="1000")
    r = subprocess.run([sys.executable, "-s", os.path.abspath(__file__), case], env=env, capture_output=True, text=True,
                       timeout=1800)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stderr[-6000:]


# ------------------------------------------------------------------------------------------------------------ cases
def _on():
    import torch
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False


def _twice(fn):
    """fn() alone, then fn() again while a large GEMM runs on another stream: the results must be identical."""
    import torch
    r1 = fn()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    big = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            big @ big
    r2 = fn()
    torch.cuda.synchronize()
    r3 = fn()
    torch.cuda.synchronize()
    for a, b, c in zip(_flat(r1), _flat(r2), _flat(r3)):
        assert torch.equal(a, b) and torch.equal(a, c)
    return r1


def _flat(r):
    return list(r) if isinstance(r, (tuple, list)) else [r]


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def case_gemm_split_k():
    import torch
    from bevbert_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(0)
    for M, N, Kd, split, bias, acc in [(256, 256, 2048, 2, False, False), (200, 136, 1000, 3, True, True),
                                       (768, 768, 8192, 4, True, True), (130, 70, 4096, 8, False, True),
                                       (1000, 768, 512, 5, True, False)]:
        a = torch.randn(M, Kd, device="cuda", generator=g).to(torch.bfloat16)
        b = torch.randn(N, Kd, device="cuda", generator=g).to(torch.bfloat16)
        bv = torch.randn(N, device="cuda", generator=g) if bias else None
        d0 = torch.randn(M, N, device="cuda", generator=g) if acc else torch.zeros(M, N, device="cuda")

        def run():
            out = d0.clone()
            K.gemm(a, b, out, M, N, Kd, lda=Kd, ldb=Kd, ldd=N, bias=bv, accumulate=acc, split_k=split)
            return out
        out = _twice(run)
        ref = d0.double() + a.double() @ b.double().t() + (bv.double() if bias else 0)
        err = float((out.double() - ref).abs().max() / ref.abs().max())
        print("gemm M=%d N=%d K=%d split=%d: max err %.2e" % (M, N, Kd, split, err))
        assert err < 1e-5, err


def case_row_reductions():
    import torch
    from bevbert_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(1)
    rows, H = 5000, 768
    x = torch.randn(rows, H, device="cuda", generator=g).to(torch.bfloat16)
    dy = torch.randn(rows, H, device="cuda", generator=g).to(torch.bfloat16)
    gamma = torch.rand(H, device="cuda", generator=g) + 0.5
    beta = torch.randn(H, device="cuda", generator=g)
    _, _, mean, rstd = K.layernorm_fwd(x, None, gamma, beta, 1e-12)

    def ln():
        dg, db, dxs = (torch.zeros(H, device="cuda") for _ in range(3))
        dx, _ = K.layernorm_bwd(dy, x, None, gamma, mean, rstd, dgamma=dg, dbeta=db, dxsum=dxs)
        return dx, dg, db, dxs
    dx, dg, db, dxs = _twice(ln)
    xh = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    assert _rel(dg, (dy.double() * xh).sum(0)) < 1e-5
    assert _rel(db, dy.double().sum(0)) < 1e-5
    assert _rel(dxs, dx.double().sum(0)) < 1e-2      # dx is stored in bf16; dxsum sums the fp32 values
    wide = torch.randn(3000, 3072, device="cuda", generator=g).to(torch.bfloat16)
    cs = _twice(lambda: K.colsum(wide, 3072))
    assert _rel(cs, wide.double().sum(0)) < 1e-5
    # unfused softmax backward with the graph bias gradient (summed over heads)
    B, Hh, nq, nk, ld = 2, 12, 20, 20, 24
    probs = torch.softmax(torch.randn(B, Hh, nq, ld, device="cuda", generator=g), -1).to(torch.bfloat16)
    dprobs = torch.randn(B, Hh, nq, ld, device="cuda", generator=g)

    def sm():
        dbias = torch.zeros(B, nq, nk, device="cuda")
        ds = K.softmax_bwd(probs, dprobs, B, Hh, nq, nk, ld, (0, 0, 1.0), 0.125, dbias)
        return ds, dbias
    _, dbias = _twice(sm)
    p, gp = probs.double()[..., :nk], dprobs.double()[..., :nk]
    ref = (p * (gp - (p * gp).sum(-1, keepdim=True))).sum(1)
    assert _rel(dbias, ref) < 1e-5


def case_scatter_exact():
    """The scatter family equals a CPU fp32 sum in ascending source order bit for bit."""
    import torch
    from bevbert_b200 import kernels as K
    g = torch.Generator().manual_seed(2)
    H = 768

    def cpu_scatter(terms, dst, nout):
        out = torch.zeros(nout, H)
        acc = {}
        for e in range(dst.numel()):
            d = int(dst[e])
            if d < 0:
                continue
            acc[d] = terms[e].clone() if d not in acc else acc[d] + terms[e]
        for d, v in acc.items():
            out[d] = out[d] + v
        return out

    # embedding gradient: repeated ids and padding_idx 0
    Bn, L, V = 6, 40, 50
    ids = torch.randint(0, V, (Bn, L), generator=g)
    ids[:, -5:] = 0
    dz = torch.randn(Bn * L, H, generator=g)
    idc, dzc = ids.cuda(), dz.cuda()

    def emb():
        dword, dpos, dtype0 = torch.zeros(V, H, device="cuda"), torch.zeros(L, H, device="cuda"), torch.zeros(H, device="cuda")
        K.embed_scatter_grad(idc, dzc, L, 0, dword, dpos, dtype0)
        return dword, dpos, dtype0
    dword, dpos, dtype0 = _twice(emb)
    flat = ids.reshape(-1)
    assert torch.equal(dword.cpu(), cpu_scatter(dz, torch.where(flat == 0, -1, flat), V))
    pos = dz.view(Bn, L, H)[0].clone()
    for b in range(1, Bn):
        pos = pos + dz.view(Bn, L, H)[b]
    assert torch.equal(dpos.cpu(), torch.zeros(L, H) + pos)
    assert _rel(dtype0, dz.double().sum(0)) < 1e-6
    # adjoint of a row gather: repeated and negative indices
    n, nout = 500, 64
    idx = torch.randint(-3, nout, (n,), generator=g)
    src = torch.randn(n, H, generator=g).to(torch.bfloat16)
    sc, ic = src.cuda(), idx.cuda()
    out = _twice(lambda: K.scatter_add_rows(sc, ic, H, torch.zeros(nout, H, device="cuda")))
    assert torch.equal(out.cpu(), cpu_scatter(src.float(), idx, nout))
    # segment weighted sum backward: overlapping segments (a source row feeds several segments)
    nseg, nsrc = 30, 40
    counts = torch.randint(0, 9, (nseg,), generator=g)
    seg_off = torch.cat([torch.zeros(1, dtype=torch.int64), counts.cumsum(0)]).to(torch.int32)
    ne = int(seg_off[-1])
    sidx = torch.randint(0, nsrc, (ne,), generator=g).to(torch.int32)
    w = torch.rand(ne, generator=g)
    dout = torch.randn(nseg, H, generator=g).to(torch.bfloat16)
    soc, sic, wc, doc = seg_off.cuda(), sidx.cuda(), w.cuda(), dout.cuda()
    dsrc = _twice(lambda: K.segment_wsum_bwd(doc, soc, sic, wc, nseg, H, torch.zeros(nsrc, H, device="cuda")))
    seg = torch.repeat_interleave(torch.arange(nseg), counts)
    terms = w[:, None] * dout.float()[seg]
    assert torch.equal(dsrc.cpu(), cpu_scatter(terms, sidx.long(), nsrc))


def case_graph_bias():
    import torch
    from bevbert_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(3)
    B, H, n = 4, 12, 20
    q, k, v, do = (torch.randn(B, n, H * 64, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4))
    bias = torch.randn(B, n, n, device="cuda", generator=g)
    o, lse = K.flash_fwd(q, k, v, B, H, n, n, H * 64, H * 64, H * 64, bias=bias)

    def bwd():
        db = torch.zeros(B, n, n, device="cuda")
        dq, dk, dv = K.flash_bwd(q, k, v, o, lse, do, B, H, n, n, H * 64, H * 64, H * 64, bias=bias, dbias=db)
        return dq, dk, dv, db
    db = _twice(bwd)[3]
    qh, kh, vh = (t.double().view(B, n, H, 64).transpose(1, 2) for t in (q, k, v))
    b64 = bias.double().requires_grad_(True)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * 0.125 + b64[:, None], -1)
    ((p @ vh) * do.double().view(B, n, H, 64).transpose(1, 2)).sum().backward()
    err = _rel(db, b64.grad)
    print("flash graph-bias gradient rel err %.2e" % err)
    assert err < 2e-2


def case_mt_sumsq():
    import torch
    from bevbert_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(4)
    sizes = [768 * 768, 3072, 30522 * 768 // 7, 5]
    ps = [torch.randn(n, device="cuda", generator=g) for n in sizes]
    gs = [torch.randn(n, device="cuda", generator=g) for n in sizes]
    rows = [(p.data_ptr(), gr.data_ptr(), 0, 0, 0, p.numel(), 0.0, 0.0) for p, gr in zip(ps, gs)]
    tab = K.MtTable(rows, "cuda")
    s = _twice(lambda: K.mt_sumsq(tab, torch.empty(1, device="cuda")).clone())
    ref = sum(float((gr.double() ** 2).sum()) for gr in gs)
    assert abs(float(s) - ref) / ref < 1e-5


def _train_setup(drop):
    from helpers import small_config
    from bevbert_b200 import synth
    from bevbert_b200.model.pretrain_cmt import GlocalTextPathCMTPreTraining
    from bevbert_b200.optim import AdamW, build_param_groups
    cfg = small_config(hidden_dropout_prob=drop, attention_probs_dropout_prob=drop, feat_dropout=0.0)
    model = synth.det_init_(GlocalTextPathCMTPreTraining(cfg), seed=3).cuda().train()
    opt = AdamW(build_param_groups(model, 0.01), lr=1e-4, betas=(0.9, 0.98), max_grad_norm=5.0, runtime=model.rt)
    return model, opt


def _train_batches():
    from helpers import small_synth
    from bevbert_b200 import synth
    from bevbert_b200.model.ops import prepare_batch
    return {t: synth.batch_to(prepare_batch(synth.make_batch(small_synth(), seed=40 + i, task=t)), "cuda")
            for i, t in enumerate(["mlm", "sap", "masksem"])}


def _train(seq, drop=0.1, side=False, graphed=False):
    import torch
    from bevbert_b200.graphs import GraphedTrainStep
    from bevbert_b200.parallel import direct_param_grads, enable_side_stream
    torch.manual_seed(0)
    b = _train_batches()
    m, o = _train_setup(drop)
    direct_param_grads(True)
    enable_side_stream(side)
    try:
        if graphed:
            step = GraphedTrainStep(m, o, warmup=1)
            losses = [step(b[t], t).detach().clone() for t in seq]
        else:
            losses = []
            for t in seq:
                loss = m(b[t], t).mean()
                loss.backward()
                o.step()
                losses.append(loss.detach().clone())
        torch.cuda.synchronize()
    finally:
        enable_side_stream(False)
        direct_param_grads(False)
    return torch.stack(losses), {n: p.detach().clone() for n, p in m.named_parameters()}


def _same(r1, r2):
    import torch
    assert torch.equal(r1[0], r2[0]), (r1[0], r2[0])
    bad = [n for n in r1[1] if not torch.equal(r1[1][n], r2[1][n])]
    assert not bad, bad[:10]


def case_train_steps():
    seq = ["mlm", "sap", "masksem", "mlm", "sap", "masksem"]
    a = _train(seq)
    _same(a, _train(seq))
    _same(a, _train(seq, side=True))
    print("losses", a[0].tolist())


def case_graph_replay():
    seq = ["mlm", "sap", "mlm", "sap", "mlm", "sap"]
    e = _train(seq, drop=0.0)
    gr = _train(seq, drop=0.0, graphed=True)
    print("eager", e[0].tolist())
    print("graph", gr[0].tolist())
    _same(e, gr)


def case_oracle_bars():
    import test_model_gpu
    for task in ("mlm", "sap", "masksem"):
        test_model_gpu.test_small_config_matches_oracle(task)


def case_nav_step():
    import torch
    from bevbert_b200 import synth
    from bevbert_b200.model.nav_vilmodel import GlocalTextPathNavCMT
    from test_nav_api_cpu import nav_batches, nav_config

    def run():
        cfg = nav_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
        model = synth.det_init_(GlocalTextPathNavCMT(cfg), seed=4).cuda().train()
        lang, _, nav = nav_batches(B=3, G=12, K=4, D=11)
        lang = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in lang.items()}
        nav = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in nav.items()}
        nav["txt_embeds"] = model("language", lang)
        fl = model("navigation", nav)["fused_logits"]
        fl[torch.isfinite(fl)].sum().backward()
        torch.cuda.synchronize()
        return {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    a, b = run(), run()
    assert a and set(a) == set(b)
    bad = [n for n in a if not torch.equal(a[n], b[n])]
    assert not bad, bad[:10]


def case_fused_scores_raises():
    import torch
    from bevbert_b200 import kernels as K
    B, H, n, ld = 2, 2, 16, 16
    t = torch.randn(B, n, H * 64, device="cuda").to(torch.bfloat16)
    P, _ = K.attn_scores_fwd(t, H * 64, t, H * 64, B, H, n, n, 64, ld, None, None, (0, 0, 1.0))
    dbias = torch.zeros(B, n, n, device="cuda")
    try:
        K.attn_scores_bwd(t, H * 64, t, H * 64, P, B, H, n, n, 64, ld, (0, 0, 1.0), dbias)
    except RuntimeError as e:
        assert "BB_FUSED_SCORES_MAX" in str(e), e
    else:
        raise AssertionError("the fused-scores graph-bias gradient ran under torch.use_deterministic_algorithms(True)")
    torch.use_deterministic_algorithms(True, warn_only=True)
    import warnings
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        K.attn_scores_bwd(t, H * 64, t, H * 64, P, B, H, n, n, 64, ld, (0, 0, 1.0), dbias)
    assert any("BB_FUSED_SCORES_MAX" in str(x.message) for x in w)
    torch.cuda.synchronize()


if __name__ == "__main__":
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    _on()
    globals()["case_" + sys.argv[1]]()
    print("ok", sys.argv[1])
