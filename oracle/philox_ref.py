"""Executable specification of the device noise of csrc/optim.cu (`fill_exponential`, `fill_normal`): Philox4x32-10
in numpy, the uniforms exactly as the kernels form them, and float64 transforms with first-order error bounds.

Layout (the kernels'): block i of four outputs is Philox4x32-10 of the counter {i & 0xffffffff, i >> 32, stream_id,
device counter} under the key {seed & 0xffffffff, seed >> 32}; the key is bumped by (0x9E3779B9, 0xBB67AE85) after
each of the ten rounds; output element 4 i + j takes word j.

Uniforms (w a 32-bit word; w >> 8 and the products below are exact in fp32 and float64):
  - exponential: u = ((w >> 8) + 1) 2^-24 in (0, 1];
  - normal: u1 = ((w_j >> 8) + 1) 2^-24 in (0, 1] and u2 = (w_{j+1} >> 8) 2^-24 in [0, 1) for the pair (j, j + 1).
Transforms:
  - exponential: max(-ln u, 1e-20);
  - normal (Box-Muller): r cos(2 pi u2) and r sin(2 pi u2), r = sqrt(-2 ln u1).
Bounds from the CUDA Math API's documented maximum errors: logf 1 ulp (at most 2u relative, u = 2^-24), sqrtf
correctly rounded (the library is not built with fast-math), sincospif 1 ulp; the product 2 u2, the factor -2 and the
negation are exact.  So the exponential is within 2u |ln u| and a normal within 5u |out| (r: u from logf through the
square root plus u from sqrtf; 2u from sincospif; u from the product).  Each bound is SAFETY times that.

Known properties, documented rather than defects:
  - the exponential's floor: u = 1 gives -ln 1 = 0, stored as 1e-20f so that p / E stays finite;
  - both samplers are truncated by the 24-bit grid: the exponential at -ln 2^-24 = 16.64, the normal at
    sqrt(2 ln 2^24) = 5.77 sigma (the normal tail beyond it has mass ~8e-9).
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24
SAFETY = 2.0
TINY = 2.0 ** -126
EXP_FLOOR = float(np.float32(1e-20))
EXP_MAX = -math.log(2.0 ** -24)                 # 16.635...
NORMAL_MAX = math.sqrt(-2.0 * math.log(2.0 ** -24))   # 5.768...

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def _mulhilo(a: int, b: np.ndarray):
    p = np.uint64(a) * b
    return p >> np.uint64(32), p & np.uint64(MASK)


def philox4x32_10(ctr, key, rounds: int = 10, bump_first: bool = False):
    """Philox4x32 of counters ctr = (c0, c1, c2, c3) (arrays or ints, broadcast) under key (k0, k1).
    bump_first bumps the key before each round instead of after it (a defect, kept for the tests)."""
    c = [np.asarray(v, dtype=np.uint64) & np.uint64(MASK) for v in ctr]
    c = list(np.broadcast_arrays(*c))
    k0, k1 = np.uint64(key[0] & MASK), np.uint64(key[1] & MASK)
    m = np.uint64(MASK)
    for _ in range(rounds):
        if bump_first:
            k0, k1 = (k0 + np.uint64(W0)) & m, (k1 + np.uint64(W1)) & m
        hi0, lo0 = _mulhilo(M0, c[0])
        hi1, lo1 = _mulhilo(M1, c[2])
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        if not bump_first:
            k0, k1 = (k0 + np.uint64(W0)) & m, (k1 + np.uint64(W1)) & m
    return np.stack(c, -1).astype(np.uint32)


def words(n: int, seed: int, stream_id: int, counter: int = 0, start: int = 0, mutant: str = None) -> np.ndarray:
    """the n uint32 words behind output elements start .. start + n - 1"""
    i = np.arange(start // 4, (start + n + 3) // 4, dtype=np.uint64)
    lo, hi = i & np.uint64(MASK), i >> np.uint64(32)
    stream, ctr = np.uint64(stream_id & MASK), np.uint64(counter & MASK)
    if mutant == "stream_counter_swapped":
        stream, ctr = ctr, stream
    w = philox4x32_10((lo, hi, stream, ctr), (seed & MASK, seed >> 32), bump_first=mutant == "key_bumped_first")
    return w.reshape(-1)[start % 4:start % 4 + n]


def exp_uniform(w: np.ndarray, mutant: str = None) -> np.ndarray:
    """u = ((w >> 8) + 1) 2^-24 in (0, 1] (float64, exact)"""
    k = (w >> np.uint32(8)).astype(np.float64)
    return (k if mutant == "u_half_open" else k + 1.0) * U


def normal_uniforms(w: np.ndarray):
    """(u1, u2) of each pair of words (elements 4i, 4i+1 from words 0, 1; 4i+2, 4i+3 from words 2, 3)"""
    w = w.reshape(-1, 2)
    return ((w[:, 0] >> np.uint32(8)).astype(np.float64) + 1.0) * U, (w[:, 1] >> np.uint32(8)).astype(np.float64) * U


def exponential(n: int, seed: int, stream_id: int, counter: int = 0, start: int = 0, mutant: str = None):
    """(value, bound, u) of fill_exponential's elements start .. start + n - 1, float64"""
    u = exp_uniform(words(n, seed, stream_id, counter, start, mutant), mutant)
    e = -np.log(u)
    v = np.maximum(e, EXP_FLOOR)
    return v, SAFETY * 2 * U * e + TINY, u


def _cospi_sinpi(x: np.ndarray):
    """cos(pi x), sin(pi x) for x in [0, 2), exact at the multiples of 1/2 (sincospif's zeros are exact there)"""
    c, s = np.cos(np.pi * x), np.sin(np.pi * x)
    h = 2 * x
    exact = h == np.round(h)
    q = np.round(h).astype(np.int64) % 4
    c = np.where(exact, np.array([1.0, 0.0, -1.0, 0.0])[q], c)
    s = np.where(exact, np.array([0.0, 1.0, 0.0, -1.0])[q], s)
    return c, s


def normal(n: int, seed: int, stream_id: int, counter: int = 0, start: int = 0, mutant: str = None):
    """(value, bound, u1, u2) of fill_normal's elements start .. start + n - 1, float64 (u1, u2 per element)"""
    first = start - start % 2                       # the pair's first element; the last pair's u2 word is read even
    count = n + start % 2                           # when its element lies past n
    u1, u2 = normal_uniforms(words(count + count % 2, seed, stream_id, counter, first, mutant))
    r = np.sqrt(-2.0 * np.log(u1))
    c, s = _cospi_sinpi(2.0 * u2)
    if mutant == "cos_sin_swapped":
        c, s = s, c
    v = np.stack([r * c, r * s], -1).reshape(-1)[start % 2:start % 2 + n]
    b = SAFETY * 5 * U * np.abs(v) + TINY
    return v, b, np.repeat(u1, 2)[start % 2:start % 2 + n], np.repeat(u2, 2)[start % 2:start % 2 + n]


def find_counter(seed: int, stream_id: int, element: int, word_pred, limit: int = 1 << 22, chunk: int = 1 << 20):
    """the smallest device counter whose word for `element` satisfies word_pred (vectorised over counters)"""
    i, j = element // 4, element % 4
    for c0 in range(0, limit, chunk):
        ctr = np.arange(c0, min(limit, c0 + chunk), dtype=np.uint64)
        w = philox4x32_10((np.uint64(i & MASK), np.uint64(i >> 32), np.uint64(stream_id), ctr),
                          (seed & MASK, seed >> 32))[:, j]
        hit = np.nonzero(word_pred(w))[0]
        if hit.size:
            return int(ctr[hit[0]])
    return None
