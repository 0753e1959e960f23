"""Times the HBM-bound kernels (BEV scatter-pool, LayerNorm fwd/bwd, column sums, casts) at the shapes of the bench
step (BASELINE configs[1]: B=32, 12x14x14 points x 768, 21x21 cells; 14112 = 32*441 token rows of 768) and prints
achieved GB/s of the ALGORITHMIC bytes against MEASURED_PEAKS.json hbm_gbs when present, else the H100 SXM data-sheet
HBM3 bandwidth (3350 GB/s).  HBM_ONLY=<name prefix> times one kernel."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bevbert_b200.kernels as K

BF = torch.bfloat16
ONLY = os.environ.get("HBM_ONLY")
PEAK, PEAK_SRC = 3350.0, "H100 SXM data sheet"
try:
    PEAK = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
    PEAK_SRC = "MEASURED_PEAKS.json"
except Exception:
    pass
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timeit(fn, n=10):
    if ONLY:
        fn()
        torch.cuda.synchronize()
        return 1.0
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(n):
        flush.zero_()     # 256 MB > 50 MB L2: every timed launch starts cold
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / n * 1e3


def report(name, us, nbytes):
    gbs = nbytes / us / 1e3
    print("%-34s %8.1f us  %7.1f MB  %7.0f GB/s  frac %.2f of %.0f (%s)" % (name, us, nbytes / 1e6, gbs, gbs / PEAK, PEAK, PEAK_SRC))


def want(name):
    return not ONLY or name.startswith(ONLY)


B, P, C, D = 32, 2352, 768, 21
ncell = D * D
g = torch.Generator(device="cuda").manual_seed(1)
if want("scatter"):
    feats = torch.randn(B, P, C, device="cuda", generator=g)
    idx = torch.randint(-60, ncell, (B, P), device="cuda", generator=g, dtype=torch.int64).clamp_(min=-1).to(torch.int32)
    t = timeit(lambda: K.bev_scatter_mean(feats, idx, ncell))
    report("scatter_mean f32 (B32,2352,768)", t, B * (P * C * 4 + P * 4 + ncell * C * 6 + ncell * 5))
    f16 = feats.to(BF)
    t = timeit(lambda: K.bev_scatter_mean(f16, idx, ncell))
    report("scatter_mean bf16 wire", t, B * (P * C * 2 + P * 4 + ncell * C * 6 + ncell * 5))
    sems = torch.nn.functional.one_hot(torch.randint(0, 40, (B, P), device="cuda", generator=g), 40).double()
    t = timeit(lambda: K.bev_scatter_sem(sems, idx, ncell))
    report("scatter_sem f64 (B32,2352,40)", t, B * (P * 40 * 8 + P * 4 + ncell * 40 * 8 + ncell))

rows, H = B * ncell, 768
if want("layernorm") or want("colsum") or want("cast"):
    x = (torch.randn(rows, H, device="cuda", generator=g)).to(BF)
    res = (torch.randn(rows, H, device="cuda", generator=g)).to(BF)
    gamma = torch.ones(H, device="cuda")
    beta = torch.zeros(H, device="cuda")
    th, sc = K.drop_params(0.1)
    drop = (5, th, sc)
if want("layernorm"):
    t = timeit(lambda: K.layernorm_fwd(x, res, gamma, beta, 1e-12, drop_in=drop))
    report("layernorm_fwd 14112x768 (+res,drop)", t, rows * (H * 2 * 3 + 8))
    y, _, mean, rstd = K.layernorm_fwd(x, res, gamma, beta, 1e-12, drop_in=drop)
    dy = (torch.randn(rows, H, device="cuda", generator=g)).to(BF)
    dg, db, dxs = (torch.zeros(H, device="cuda") for _ in range(3))
    t = timeit(lambda: K.layernorm_bwd(dy, x, res, gamma, mean, rstd, drop_in=drop, want_dres=True, dgamma=dg, dbeta=db,
                                       dxsum=dxs))
    report("layernorm_bwd 14112x768 (+dres)", t, rows * (H * 2 * 5 + 8))
if want("colsum"):
    w = (torch.randn(rows, 3 * H, device="cuda", generator=g)).to(BF)
    out = torch.zeros(3 * H, device="cuda")
    t = timeit(lambda: K.colsum(w, 3 * H, out=out))
    report("colsum 14112x2304", t, rows * 3 * H * 2)
if want("cast"):
    w32 = torch.randn(3072, 768, device="cuda", generator=g)
    w16 = torch.empty(3072, 768, dtype=BF, device="cuda")
    t = timeit(lambda: K.cast_to_act(w32, out=w16))
    report("cast f32->bf16 3072x768", t, 3072 * 768 * 6)
    big = torch.randn(rows, H, device="cuda", generator=g)
    t = timeit(lambda: K.cast_to_act(big, drop))
    report("cast+dropout f32->bf16 14112x768", t, rows * H * 6)
