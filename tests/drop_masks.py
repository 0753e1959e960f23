"""Exact torch restatements of the dropout decision functions of the CUDA kernels (test infrastructure).

Every function returns a bool keep mask computed with int64 tensors that wrap mod 2^32 exactly like the uint32
arithmetic of the kernels; products are split into 16-bit halves so that no int64 product can overflow.  `seed` is
the 64-bit site seed (blocks.DropState gives seeds >= 2^63) and `salt` the graph-replay salt the kernels XOR into it
(bb_set_drop_salt_ptr; 0 = no salt registered).

- keep_elem: one full hash per element index (csrc/ptx.cuh rng_u32 / drop_keep).  GEMM epilogues (index = element
  offset in D, batch offset included), bb_cast_f32_bf16, bb_dropout_bf16, the fp32-arm GEMM.
- ln_keep: the LayerNorm sites (csrc/rowops.cu ln_keep8): one hash per 8-element vector, four mixes whose 16-bit
  halves decide two elements each.
- attn_keep: the fused attention probabilities (csrc/attn_flash.cu, csrc/attn_tc.cu): one hash per (sample, head,
  query) row, one mix per pair of adjacent keys, low 16 bits for the even key, high 16 bits for the odd key.
- softmax_keep: the unfused / fused-scores probabilities (bb_softmax_fwd / _bwd, bb_attn_scores): keep_elem at
  row * ld + key.
The 16-bit sites compare against thresh & 0xFFFF0000.
"""
import torch

M32 = 0xFFFFFFFF
_U64 = (1 << 64) - 1


def _mul32(x, c):
    """(x * c) mod 2^32 for int64 tensors x in [0, 2^32) and a Python constant c < 2^32, without int64 overflow."""
    return (x * (c & 0xFFFF) + (((x * (c >> 16)) & 0xFFFF) << 16)) & M32


def _seed_word(seed, salt):
    """the 32-bit seed term of rng_u32 (a Python int)"""
    s = (int(seed) ^ int(salt)) & _U64
    return (s & M32) ^ (((s >> 32) * 0x85EBCA6B) & M32)


def rng_u32(seed, idx, salt=0):
    """32 random bits of (seed ^ salt, idx); idx: int64 tensor of non-negative element indices."""
    idx = torch.as_tensor(idx, dtype=torch.int64)
    x = (idx & M32) ^ _mul32((idx >> 32) & M32, 0x9E3779B1) ^ _seed_word(seed, salt)
    x = x ^ (x >> 16)
    x = _mul32(x, 0x7FEB352D)
    x = x ^ (x >> 15)
    x = _mul32(x, 0x846CA68B)
    return x ^ (x >> 16)


def keep_elem(seed, idx, thresh, salt=0):
    return rng_u32(seed, idx, salt) >= int(thresh)


def _mix(h, k):
    """one multiply-xorshift round on a Weyl step of a 32-bit hash (the pair / vector mixes of the 16-bit sites)"""
    x = (h + _mul32(torch.as_tensor(k, dtype=torch.int64), 0x9E3779B1)) & M32
    x = x ^ (x >> 15)
    x = _mul32(x, 0x2C1B3C6D)
    return x ^ (x >> 16)


def _half_keep(x, odd, thresh):
    t16s = int(thresh) & 0xFFFF0000
    return torch.where(odd, x, (x << 16) & M32) >= t16s


def ln_keep_vec(seed, vec, thresh, salt=0):
    """(n, 8) keep mask of the 8-element vectors with indices `vec` (element index >> 3)."""
    h = rng_u32(seed, vec, salt)[:, None]
    j = torch.arange(8, dtype=torch.int64)
    return _half_keep(_mix(h, (j >> 1) + 1), (j & 1).bool(), thresh)


def ln_keep(seed, rows, H, thresh, salt=0):
    """(rows, H) keep mask of a LayerNorm site over a row-major (rows, H) tensor, H % 8 == 0."""
    assert H % 8 == 0
    return ln_keep_vec(seed, torch.arange(rows * H // 8, dtype=torch.int64), thresh, salt).reshape(rows, H)


def attn_keep_rows(seed, rows, keys, thresh, salt=0):
    """(len(rows), len(keys)) keep mask of the fused attention sites; rows = (b * H + h) * nq + q."""
    rh = rng_u32(seed, rows, salt)[:, None]
    keys = torch.as_tensor(keys, dtype=torch.int64)[None, :]
    return _half_keep(_mix(rh, keys >> 1), (keys & 1).bool(), thresh)


def attn_keep(seed, B, H, nq, nk, thresh, salt=0):
    """(B, H, nq, nk) keep mask of the attention probabilities in bb_flash_fwd / bb_flash_bwd."""
    return attn_keep_rows(seed, torch.arange(B * H * nq, dtype=torch.int64), torch.arange(nk), thresh,
                          salt).reshape(B, H, nq, nk)


def softmax_keep(seed, B, H, nq, nk, ld, thresh, salt=0):
    """(B, H, nq, nk) keep mask of the probabilities in bb_softmax_fwd / _bwd and bb_attn_scores (row stride ld)."""
    rows = torch.arange(B * H * nq, dtype=torch.int64)[:, None]
    return keep_elem(seed, rows * ld + torch.arange(nk, dtype=torch.int64)[None, :], thresh, salt).reshape(B, H, nq, nk)
