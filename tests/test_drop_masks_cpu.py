"""The vectorised mask restatements of tests/drop_masks.py against a plain scalar transcription of the kernels' uint32
code (explicit & 0xFFFFFFFF after every step), over seeds >= 2^63, element indices >= 2^32 and thresholds whose low
16 bits are nonzero."""
import random

import torch

import drop_masks as DM

M = 0xFFFFFFFF


def s_rng(seed, idx):
    seed &= (1 << 64) - 1
    x = (idx & M) ^ (((idx >> 32) * 0x9E3779B1) & M) ^ (seed & M) ^ (((seed >> 32) * 0x85EBCA6B) & M)
    x ^= x >> 16
    x = (x * 0x7FEB352D) & M
    x ^= x >> 15
    x = (x * 0x846CA68B) & M
    x ^= x >> 16
    return x


def s_mix(h, k):
    x = (h + k * 0x9E3779B1) & M
    x ^= x >> 15
    x = (x * 0x2C1B3C6D) & M
    x ^= x >> 16
    return x


def s_ln_keep(seed, elem, thresh):
    x = s_mix(s_rng(seed, elem >> 3), ((elem & 7) >> 1) + 1)
    half = (x >> 16) if elem & 1 else (x & 0xFFFF)
    return half >= (thresh >> 16)


def s_attn_keep(seed, row, k, thresh):
    x = s_mix(s_rng(seed, row), k >> 1)
    half = (x >> 16) if k & 1 else (x & 0xFFFF)
    return half >= (thresh >> 16)


SEEDS = [0, 1, 0x12345678, 0xFFFFFFFF, 1 << 32, 0x9E3779B97F4A7C15, 0xFFFFFFFFFFFFFFFF, (1 << 63) | 0x5A5A]
THRESHES = [0x19999999, 0x80000001, 0x0000FFFF, 0xFFFF0000, 0xCCCCCCCC]


def _indices(rng, n=3000):
    idx = list(range(40)) + [(1 << 32) - 1, 1 << 32, (1 << 32) + 7, (1 << 40) + 3, (1 << 62) + 11]
    idx += [rng.randrange(0, 1 << 24) for _ in range(n // 2)] + [rng.randrange(1 << 32, 1 << 62) for _ in range(n // 2)]
    return idx


def test_rng_u32_and_keep_elem_match_scalar_code():
    rng = random.Random(0)
    idx = _indices(rng)
    t = torch.tensor(idx, dtype=torch.int64)
    for seed in SEEDS:
        for salt in (0, 0x2545F4914F6CDD1D):
            got = DM.rng_u32(seed, t, salt)
            assert got.tolist() == [s_rng(seed ^ salt, i) for i in idx]
            th = THRESHES[seed % len(THRESHES)]
            assert DM.keep_elem(seed, t, th, salt).tolist() == [s_rng(seed ^ salt, i) >= th for i in idx]


def test_ln_keep_matches_scalar_code():
    rng = random.Random(1)
    vec = [v >> 3 for v in _indices(rng, 1000)]
    t = torch.tensor(vec, dtype=torch.int64)
    for seed, th in zip(SEEDS, THRESHES * 2):
        for salt in (0, 0x0DDB1A5E5BAD5EED):
            got = DM.ln_keep_vec(seed, t, th, salt)
            ref = [[s_ln_keep(seed ^ salt, v * 8 + j, th) for j in range(8)] for v in vec]
            assert got.tolist() == ref
    # the (rows, H) form: element (r, c) is element r * H + c of the flat tensor
    rows, H = 5, 24
    got = DM.ln_keep(SEEDS[5], rows, H, THRESHES[0])
    assert got.tolist() == [[s_ln_keep(SEEDS[5], r * H + c, THRESHES[0]) for c in range(H)] for r in range(rows)]


def test_attn_keep_matches_scalar_code():
    rng = random.Random(2)
    rows = [0, 1, (1 << 32) - 1, 1 << 32, (1 << 33) + 5] + [rng.randrange(0, 1 << 40) for _ in range(45)]
    keys = list(range(70)) + [441, 510, 511]
    for seed, th in zip(SEEDS, THRESHES * 2):
        for salt in (0, 0x0DDB1A5E5BAD5EED):
            got = DM.attn_keep_rows(seed, torch.tensor(rows), torch.tensor(keys), th, salt)
            assert got.tolist() == [[s_attn_keep(seed ^ salt, r, k, th) for k in keys] for r in rows]
    B, H, nq, nk = 2, 3, 5, 7
    got = DM.attn_keep(SEEDS[6], B, H, nq, nk, THRESHES[0])
    ref = [[[[s_attn_keep(SEEDS[6], (b * H + h) * nq + q, k, THRESHES[0]) for k in range(nk)] for q in range(nq)]
            for h in range(H)] for b in range(B)]
    assert got.tolist() == ref


def test_softmax_keep_matches_scalar_code():
    B, H, nq, nk, ld = 2, 3, 17, 21, 24
    for seed, th in zip(SEEDS, THRESHES * 2):
        for salt in (0, 0x0DDB1A5E5BAD5EED):
            got = DM.softmax_keep(seed, B, H, nq, nk, ld, th, salt)
            ref = [[[[s_rng(seed ^ salt, ((b * H + h) * nq + q) * ld + k) >= th for k in range(nk)] for q in range(nq)]
                    for h in range(H)] for b in range(B)]
            assert got.tolist() == ref


def test_sixteen_bit_sites_ignore_the_low_threshold_bits():
    """thresh 0x1999_9999 (p = 0.1) at the 16-bit sites is compared as 0x1999_0000: a half equal to 0x1999 is kept"""
    seed, vec = SEEDS[5], torch.arange(4096, dtype=torch.int64)
    a = DM.ln_keep_vec(seed, vec, 0x19999999)
    b = DM.ln_keep_vec(seed, vec, 0x19990000)
    assert torch.equal(a, b)
    assert abs(float(a.float().mean()) - 0.9) < 0.01
