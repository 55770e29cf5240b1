"""numpy restatements of the contracts of csrc/rng.cu (include/lidiff_b200.h, host random streams), step for step:
the three-phase MT19937 twist on two buffers, the legacy Gaussian's attempt / scan indexing, the log band classification and the
randperm reservation rounds.  Each is checked against np.random.randn / torch.randperm in test_rng_host.py."""
import math

import numpy as np

MT_N, MT_M = 624, 397
UPPER, LOWER, MATRIX_A = np.uint32(0x80000000), np.uint32(0x7FFFFFFF), np.uint32(0x9908B0DF)


def _mix(a, b, src):
    y = (a & UPPER) | (b & LOWER)
    return src ^ (y >> np.uint32(1)) ^ np.where((y & np.uint32(1)) != 0, MATRIX_A, np.uint32(0)).astype(np.uint32)


def twist_phases(a: np.ndarray) -> np.ndarray:
    """k_mt_words' twist: three vector phases from the old buffer `a` into a new one"""
    a = np.asarray(a, np.uint32)
    b = np.empty_like(a)
    d = MT_N - MT_M
    i = np.arange(d)
    b[i] = _mix(a[i], a[i + 1], a[i + MT_M])
    i = np.arange(d, 2 * d)
    b[i] = _mix(a[i], a[i + 1], b[i - d])
    i = np.arange(2 * d, MT_N - 1)
    b[i] = _mix(a[i], a[i + 1], b[i - d])
    b[MT_N - 1] = _mix(a[MT_N - 1], b[0], b[MT_M - 1])
    return b


def temper(y: np.ndarray) -> np.ndarray:
    y = np.asarray(y, np.uint32).copy()
    y ^= y >> np.uint32(11)
    y ^= (y << np.uint32(7)) & np.uint32(0x9D2C5680)
    y ^= (y << np.uint32(15)) & np.uint32(0xEFC60000)
    return y ^ (y >> np.uint32(18))


def mt_words(key: np.ndarray, pos: int, n: int):
    """(n tempered words, key after, pos after) as lb2_mt19937_words"""
    key = np.asarray(key, np.uint32).copy()
    out = []
    done = 0
    while done < n:
        if pos == MT_N:
            key, pos = twist_phases(key), 0
        take = min(MT_N - pos, n - done)
        out.append(temper(key[pos:pos + take]))
        done += take
        pos += take
    return (np.concatenate(out) if out else np.zeros(0, np.uint32)), key, pos


def attempts(words: np.ndarray):
    """(x1, x2, r2, accepted) of every 4-word attempt, in the kernel's exact operations (no FMA)"""
    w = np.asarray(words, np.uint32)[: len(words) // 4 * 4].reshape(-1, 4).astype(np.uint64)
    d1 = ((w[:, 0] >> np.uint64(5)) * np.uint64(1 << 26) + (w[:, 1] >> np.uint64(6))).astype(np.float64) * 2.0 ** -53
    d2 = ((w[:, 2] >> np.uint64(5)) * np.uint64(1 << 26) + (w[:, 3] >> np.uint64(6))).astype(np.float64) * 2.0 ** -53
    x1, x2 = 2.0 * d1 - 1.0, 2.0 * d2 - 1.0
    r2 = x1 * x1 + x2 * x2
    return x1, x2, r2, (r2 < 1.0) & (r2 != 0.0)


def midpoint_distance(r2: np.ndarray) -> np.ndarray:
    """distance (in ulp of the rounded value) of the exact log(r2) from the nearest rounding midpoint, from a long-double log
    (x86's 64-bit significand: the estimate is good to about 2^-10 ulp); nan where the rounded value is a power of two"""
    v = np.log(np.asarray(r2, np.longdouble))
    y = v.astype(np.float64)
    ulp = np.spacing(np.abs(y))
    frac = np.abs((v - y.astype(np.longdouble)) / ulp.astype(np.longdouble)).astype(np.float64)
    dist = 0.5 - frac
    mant = np.frexp(np.abs(y))[0]
    return np.where(mant == 0.5, np.nan, dist)


def deferred(r2: np.ndarray, band: float) -> np.ndarray:
    """the attempts whose log the host resolves: within `band` ulp of a midpoint (or at a power of two)"""
    d = midpoint_distance(r2)
    return ~(d > band)


def libm_log(x: np.ndarray) -> np.ndarray:
    """glibc's log element by element (math.log calls it, as numpy's legacy_gauss does; np.log is numpy's own SIMD log)"""
    return np.array([math.log(v) for v in np.asarray(x, np.float64).ravel()]).reshape(np.shape(x))


def legacy_gauss(key, pos, has_gauss, gauss, n, log=libm_log):
    """np.random.randn(n) from the state, as lb2_legacy_gauss indexes it: accepted attempt of rank r gives outputs
    hg + 2r (f x2) and hg + 2r + 1 (f x1); returns (out, key, pos, has_gauss, gauss, words used, accepted r2)"""
    hg = 1 if has_gauss else 0
    out = np.empty(n)
    if n == 0:
        return out, key, pos, has_gauss, gauss, 0, np.zeros(0)
    if hg:
        out[0] = gauss
    pairs = (n - hg + 1) // 2
    if pairs == 0:
        return out, key, pos, 0, 0.0, 0, np.zeros(0)
    nw = 4 * (2 * pairs + 64)
    while True:
        words, _, _ = mt_words(key, pos, nw)
        x1, x2, r2, acc = attempts(words)
        rank = np.cumsum(acc) - 1                      # the scan of the accept flags
        if acc.sum() >= pairs:
            break
        nw *= 2
    ks = np.flatnonzero(acc)[:pairs]
    f = np.sqrt(-2.0 * log(r2[ks]) / r2[ks])
    assert (rank[ks] == np.arange(pairs)).all()
    o = hg + 2 * np.arange(pairs)
    out[o] = f * x2[ks]
    odd = (n - hg) % 2 == 1
    last = o + 1 < n
    out[o[last] + 1] = (f * x1[ks])[last]
    used = 4 * (int(ks[-1]) + 1)
    _, key2, pos2 = mt_words(key, pos, used)
    return out, key2, pos2, int(odd), float(f[-1] * x1[ks[-1]]) if odd else 0.0, used, r2[ks]


def fisher_yates(words: np.ndarray, n: int) -> np.ndarray:
    r = np.arange(n, dtype=np.int64)
    for i in range(n - 1):
        z = int(words[i]) % (n - i)
        r[i], r[i + z] = r[i + z], r[i]
    return r


def randperm_rounds(words: np.ndarray, n: int):
    """lb2_randperm's rounds of deterministic reservations: (permutation, rounds)"""
    out = np.arange(n, dtype=np.int64)
    if n < 2:
        return out, 0
    i_all = np.arange(n - 1, dtype=np.int64)
    j_all = i_all + np.asarray(words[: n - 1], np.int64) % (n - i_all)
    res = np.full(n, np.iinfo(np.uint64).max, np.uint64)
    open_ = i_all
    r = 0
    while open_.size:
        key = np.uint64((0xFFFFFFFF - r) << 32) | open_.astype(np.uint64)   # later rounds win: stale reservations stay
        np.minimum.at(res, open_, key)
        np.minimum.at(res, j_all[open_], key)
        win = (res[open_] == key) & (res[j_all[open_]] == key)
        i, j = open_[win], j_all[open_[win]]
        out[i], out[j] = out[j].copy(), out[i].copy()
        open_ = open_[~win]
        r += 1
    return out, r
