"""Times the fused attention core (bb_flash_fwd / bb_flash_bwd) at the shapes of the bench step (B=32, 12 heads)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bevbert_b200.kernels as K

BF = torch.bfloat16
B, H, Hd = 32, 12, 768


ONLY = os.environ.get("ATTN_ONLY")


def timeit(fn, n=20):
    if ONLY:
        fn()
        torch.cuda.synchronize()
        return 1.0
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


for name, b, nq, nk, cross, p in [("bev self 441", B, 441, 441, False, 0.1), ("lang self 80", B, 80, 80, False, 0.1),
                                  ("bev->lang 441x80", B, 441, 80, True, 0.1), ("lang->bev 80x441", B, 80, 441, True, 0.1),
                                  ("gmap self 23", B, 23, 23, False, 0.1), ("gmap->lang 23x80", B, 23, 80, True, 0.1),
                                  ("pano 36 x179", 179, 36, 36, False, 0.1), ("bev self 441 p=0", B, 441, 441, False, 0.0)]:
    if ONLY and not name.startswith(ONLY):
        continue
    if not cross:
        qkv = (torch.randn(b * nq, 3 * Hd, device="cuda") * 0.5).to(BF)
        q, k, v, ldq, ldk, ldv = qkv, qkv[:, Hd:], qkv[:, 2 * Hd:], 3 * Hd, 3 * Hd, 3 * Hd
    else:
        q = (torch.randn(b * nq, Hd, device="cuda") * 0.5).to(BF)
        kv = (torch.randn(b * nk, 2 * Hd, device="cuda") * 0.5).to(BF)
        k, v, ldq, ldk, ldv = kv, kv[:, Hd:], Hd, 2 * Hd, 2 * Hd
    kmask = torch.zeros(b, nk, device="cuda")
    th, sc = K.drop_params(p)
    drop = (11, th, sc)
    o, lse = K.flash_fwd(q, k, v, b, H, nq, nk, ldq, ldk, ldv, kmask, None, drop)
    dout = (torch.randn(b, nq, Hd, device="cuda") * 0.1).to(BF)
    dq = torch.empty(b * nq, Hd, dtype=BF, device="cuda")
    dk = torch.empty(b * nk, Hd, dtype=BF, device="cuda")
    dv = torch.empty(b * nk, Hd, dtype=BF, device="cuda")
    tf = timeit(lambda: K.flash_fwd(q, k, v, b, H, nq, nk, ldq, ldk, ldv, kmask, None, drop))
    tb = timeit(lambda: K.flash_bwd(q, k, v, o, lse, dout, b, H, nq, nk, ldq, ldk, ldv, kmask, None, drop,
                                    out=(dq, Hd, dk, Hd, dv, Hd)))
    fl = 4.0 * b * H * nq * nk * 64
    print("%-20s fwd %7.1f us (%6.1f TF/s)   bwd %7.1f us (%6.1f TF/s of 3.5x fwd flops)" % (
        name, tf, fl / tf / 1e6, tb, 3.5 * fl / tb / 1e6))
