"""numpy restatements of the contracts of csrc/rng.cu (include/lidiff_b200.h, host random streams), step for step:
the three-phase MT19937 twist on two buffers, the legacy Gaussian's attempt / scan indexing, the log band classification and the
randperm reservation rounds.  Each is checked against np.random.randn / torch.randperm in test_rng_host.py.

Also the edge inputs of the device streams (test_gpu_device_rng_edges.py, checked in test_rng_reference_host.py): an exact log
oracle (`cr_log`), attempts crafted word by word (`words_for`, `pair_for_r2`, the attempt sets) and numpy states that emit given
words next (`crafted_state`)."""
import functools
import math
from decimal import Context, Decimal

import numpy as np

from lidiff_b200 import rng

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


def gauss_from_words(words: np.ndarray, n_out: int, has_gauss=0, gauss=0.0, log=libm_log):
    """lb2_legacy_gauss over the attempts of `words` (4 words each; a partial attempt is ignored): accepted attempt of rank r gives
    outputs hg + 2r (f x2) and hg + 2r + 1 (f x1), f = sqrt(-2 log(r2) / r2).  Returns (out, info): info holds the Lb2GaussInfo
    fields words_used, short_words, has_gauss, gauss, and `r2` / `k`, the r2 and attempt index of each output pair."""
    hg = 1 if has_gauss else 0
    out = np.zeros(n_out)
    info = dict(words_used=0, short_words=0, has_gauss=hg, gauss=float(gauss), r2=np.zeros(0), k=np.zeros(0, np.int64))
    if n_out == 0:
        return out, info
    if hg:
        out[0] = gauss
    pairs = (n_out - hg + 1) // 2
    if pairs == 0:                                     # the cached value alone: numpy clears the cache
        info.update(has_gauss=0, gauss=0.0)
        return out, info
    x1, x2, r2, acc = attempts(words)
    ks = np.flatnonzero(acc)[:pairs]                   # the scan of the accept flags
    if ks.size < pairs:
        info.update(short_words=1)
        return out, info
    f = np.sqrt(-2.0 * log(r2[ks]) / r2[ks])
    o = hg + 2 * np.arange(pairs)
    out[o] = f * x2[ks]
    last = o + 1 < n_out
    out[o[last] + 1] = (f * x1[ks])[last]
    odd = (n_out - hg) % 2 == 1
    info.update(words_used=4 * (int(ks[-1]) + 1), has_gauss=int(odd), gauss=float(f[-1] * x1[ks[-1]]) if odd else 0.0, r2=r2[ks],
                k=ks)
    return out, info


def legacy_gauss(key, pos, has_gauss, gauss, n, log=libm_log):
    """np.random.randn(n) from the state, as lb2_legacy_gauss indexes it (gauss_from_words over the state's words); returns
    (out, key, pos, has_gauss, gauss, words used, accepted r2)"""
    nw = 4 * (n + 64)
    while True:
        words, _, _ = mt_words(key, pos, nw)
        out, info = gauss_from_words(words, n, has_gauss, gauss, log)
        if not info["short_words"]:
            break
        nw *= 2
    _, key2, pos2 = mt_words(key, pos, info["words_used"])
    return out, key2, pos2, info["has_gauss"], info["gauss"], info["words_used"], info["r2"]


def fisher_yates(words: np.ndarray, n: int) -> np.ndarray:
    """torch's sequential shuffle: for i < n - 1, swap(r[i], r[i + words[i] % (n - i)])"""
    r = list(range(n))
    if n > 1:
        z = (np.asarray(words[: n - 1]).astype(np.uint32).astype(np.int64) % np.arange(n, 1, -1, dtype=np.int64)).tolist()
        for i, zi in enumerate(z):
            j = i + zi
            r[i], r[j] = r[j], r[i]
    return np.array(r, dtype=np.int64)


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


# ---- randperm word patterns ----------------------------------------------------------------------------------------------------
# name -> (words of n - 1 iterations, closed-form reservation rounds or None).  z_i = word_i % (n - i); an iteration closes in the
# first round in which it holds both of its slots, and the smallest open index wins every contested slot.
def _rp_small_z(n):
    return np.random.RandomState(n).randint(0, 3, n - 1).astype(np.uint32)


RANDPERM_PATTERNS = {
    "zeros": (lambda n: np.zeros(n - 1, np.uint32), lambda n: 1),                       # z = 0: nothing contested
    "last_slot": (lambda n: (n - 1 - np.arange(n - 1)).astype(np.uint32), lambda n: n - 1),   # every i aims at slot n - 1
    "chain": (lambda n: np.ones(n - 1, np.uint32), lambda n: n - 1),                     # z = 1: i waits for i - 1
    "odd_one": (lambda n: (np.arange(n - 1) & 1).astype(np.uint32), lambda n: 1 if n <= 3 else 2),   # odd i takes i + 1 first
    "even_one": (lambda n: (1 - (np.arange(n - 1) & 1)).astype(np.uint32), lambda n: 1 if n == 2 else 2),
    "all_ones": (lambda n: np.full(n - 1, 0xFFFFFFFF, np.uint32), None),
    "small_z": (_rp_small_z, None),                                                      # random z in {0, 1, 2}
}


# ---- crafted Gaussian attempts --------------------------------------------------------------------------------------------------
D_ZERO = 1 << 52                                   # the legacy 53-bit integer d of x = 0; d = D_ZERO + k gives x = k 2^-52 exactly
_M26 = (1 << 26) - 1


def words_for(d1, d2) -> np.ndarray:
    """the words whose legacy doubles are the 53-bit integers d1, d2 (x = 2 d 2^-53 - 1): 4 per attempt, flattened (uint32)"""
    d1 = np.atleast_1d(np.asarray(d1, np.int64))
    d2 = np.atleast_1d(np.asarray(d2, np.int64))
    w = np.stack([(d1 >> 26) << 5, (d1 & _M26) << 6, (d2 >> 26) << 5, (d2 & _M26) << 6], axis=-1)
    return w.astype(np.uint32).ravel()


def crafted_state(words_wanted, has_gauss=0, gauss=0.0):
    """a numpy RandomState whose next len(words_wanted) (<= 624) words are `words_wanted`: it sits at pos 624 - len with the key's
    last words untempered from them (the words after them come from twisting that key)"""
    words_wanted = np.asarray(words_wanted, np.uint32)
    assert 0 < words_wanted.size <= MT_N
    rs = np.random.RandomState(0)
    _, key, _, _, _ = rs.get_state(legacy=True)
    key = key.copy()
    pos = MT_N - words_wanted.size
    key[pos:] = rng.untemper(words_wanted)
    rs.set_state(("MT19937", key, pos, int(has_gauss), float(gauss)))
    return rs


_LN = Context(prec=60)


@functools.lru_cache(maxsize=None)
def cr_log(r2: float):
    """(the correctly rounded log(r2), the signed distance of the exact log from the nearest rounding midpoint in ulp), 0 < r2 < 1.
    The log is a 60-digit decimal (Decimal(float) is exact, float(Decimal) rounds correctly, and the exact log of a double other
    than 1 is never a midpoint).  The ulp is the gap between the rounded value and its neighbour across that midpoint (at a power
    of two, the gap on the exact value's side); the distance is positive when the exact log lies above the midpoint."""
    r2 = float(r2)
    assert 0.0 < r2 < 1.0, r2
    L = _LN.ln(Decimal(r2))
    y = float(L)
    Y = Decimal(y)
    nb = Decimal(math.nextafter(y, math.inf if L > Y else -math.inf))
    mid = _LN.divide(_LN.add(Y, nb), 2)
    return y, float(_LN.divide(_LN.subtract(L, mid), abs(_LN.subtract(nb, Y))))


def cr_logs(r2: np.ndarray):
    """cr_log over an array: (correctly rounded logs, unsigned midpoint distances in ulp)"""
    res = [cr_log(float(v)) for v in np.asarray(r2, np.float64).ravel()]
    return np.array([y for y, _ in res]), np.abs(np.array([d for _, d in res]))


def is_pow2(y: np.ndarray) -> np.ndarray:
    return np.frexp(np.abs(np.asarray(y, np.float64)))[0] == 0.5


def pair_for_r2(target: float, tries: int = 1 << 12):
    """(d1, d2) of an attempt with x1, x2 >= 0 whose r2 (the kernel's fl(fl(x1^2) + fl(x2^2))) is exactly `target`, or None: x1
    just below sqrt(target), x2 filling the rest"""
    k1 = int(math.isqrt(int(target * 2.0 ** 104))) - np.arange(tries, dtype=np.int64)
    k1 = k1[k1 >= 0]
    a = (k1 * 2.0 ** -52) ** 2
    base = np.rint(np.sqrt(np.maximum(target - a, 0.0)) * 2.0 ** 52)
    for dk in (0, -1, 1, -2, 2):
        k2 = base + dk
        hit = np.flatnonzero((k2 >= 0) & (k2 < 2.0 ** 52) & (a + (k2 * 2.0 ** -52) ** 2 == target))
        if hit.size:
            return D_ZERO + int(k1[hit[0]]), D_ZERO + int(k2[hit[0]])
    return None


def _pair_at_most(target: float):
    """(d1, d2) of a large r2 <= target: the exact target or a few ulp below it where r2 >= 2^-40 (x2 small fills what x1^2 leaves),
    else the largest k1^2 + k2^2 <= target 2^104 with k1 = isqrt, k1 stepped down while the rounded sum exceeds the target"""
    if target >= 2.0 ** -40:
        for _ in range(16):
            p = pair_for_r2(target)
            if p is not None:
                return p
            target = math.nextafter(target, 0.0)
        raise AssertionError("no attempt found below the target")
    n = int(target * 2.0 ** 104)
    k1 = math.isqrt(n)
    while True:
        p = D_ZERO + k1, D_ZERO + math.isqrt(n - k1 * k1)
        if attempts(words_for(*p))[2][0] <= target:
            return p
        k1 -= 1


def polar_edges():
    """[(name, d1, d2, accepted)]: the polar method's rejections and accepted extremes, with both signs of each coordinate"""
    lo = pair_for_r2(math.nextafter(1.0, 0.0))
    k = 1351079888211149                                # x = 0.29999999999999993...
    return [
        ("r2_zero", D_ZERO, D_ZERO, False),
        ("x1_minus_one", 0, D_ZERO, False),             # r2 = 1
        ("x2_minus_one", D_ZERO, 0, False),
        ("r2_two", 0, 0, False),
        ("r2_just_above_one", 1, D_ZERO + (1 << 27), False),      # (1 - 2^-51) + 2^-50
        ("smallest_r2", D_ZERO + 1, D_ZERO, True),      # x1 = 2^-52: r2 = 2^-104
        ("smallest_r2_x1_negative", D_ZERO - 1, D_ZERO, True),
        ("smallest_r2_x2", D_ZERO, D_ZERO + 1, True),
        ("smallest_r2_x2_negative", D_ZERO, D_ZERO - 1, True),
        ("x1_minus_one_plus_ulp", 1, D_ZERO, True),     # r2 = 1 - 2^-51
        ("largest_r2", lo[0], lo[1], True),             # r2 = 1 - 2^-53
        ("largest_r2_negative", 2 * D_ZERO - lo[0], 2 * D_ZERO - lo[1], True),
        ("x1_zero", D_ZERO, D_ZERO + (3 << 50), True),  # x2 = 0.75
        ("x1_zero_x2_negative", D_ZERO, D_ZERO - (3 << 50), True),
        ("x2_zero", D_ZERO + k, D_ZERO, True),
        ("x2_zero_x1_negative", D_ZERO - k, D_ZERO, True),
        ("quadrant_pp", D_ZERO + k, D_ZERO + 2 * k, True),
        ("quadrant_pm", D_ZERO + k, D_ZERO - 2 * k, True),
        ("quadrant_mp", D_ZERO - k, D_ZERO + 2 * k, True),
        ("quadrant_mm", D_ZERO - k, D_ZERO - 2 * k, True),
    ]


def binade_attempts():
    """(d1, d2) with r2 at the bottom (exactly 2^-j), the middle (about 1.5 2^-j) and the top (the largest found below 2^-(j-1))
    of every binade [2^-j, 2^-(j-1)), j = 1 .. 104"""
    out = []
    for j in range(1, 105):
        if j % 2 == 0:
            out.append((D_ZERO + (1 << (52 - j // 2)), D_ZERO))
        else:
            out.append((D_ZERO + (1 << (52 - (j + 1) // 2)),) * 2)
        out.append(_pair_at_most(1.5 * 2.0 ** -j))
        out.append(_pair_at_most(math.nextafter(2.0 ** -(j - 1), 0.0)))
    return tuple(np.array(c, np.int64) for c in zip(*out))


def switch_attempts(binades=(0, 1, 2, 7, 19)):
    """(d1, d2) with r2 = c 2^-j, c the double nearest 1/sqrt(2) and 8 ulp either side: dd_log's m < 0.7071... switch"""
    c0 = float(_LN.sqrt(Decimal("0.5")))
    out = []
    for j in binades:
        c = c0
        for _ in range(8):
            c = math.nextafter(c, 0.0)
        for _ in range(17):
            out.append(pair_for_r2(math.ldexp(c, -j)))
            c = math.nextafter(c, 1.0)
    return tuple(np.array(c, np.int64) for c in zip(*out))


POW2_LOGS = (-1.0, -2.0, -0.5, -0.25)


def pow2_attempts(span: int = 24):
    """(d1, d2) with r2 the double nearest exp(p) and `span` ulp either side, p in POW2_LOGS: logs at and next to powers of two"""
    out = []
    for p in POW2_LOGS:
        t = float(_LN.exp(Decimal(p)))
        for _ in range(span):
            t = math.nextafter(t, 0.0)
        for _ in range(2 * span + 1):
            out.append(pair_for_r2(t))
            t = math.nextafter(t, 1.0)
    return tuple(np.array(c, np.int64) for c in zip(*out))


def random_accepted(n: int, seed: int):
    """(d1, d2) of n accepted attempts uniform in the unit disc"""
    rs = np.random.RandomState(seed)
    d = rs.randint(0, 1 << 53, (2, 2 * n + 64), dtype=np.int64)
    _, _, _, acc = attempts(words_for(d[0], d[1]))
    return d[0][acc][:n], d[1][acc][:n]


def random_rejected(n: int, seed: int):
    """(d1, d2) of n rejected attempts: the crafted rejections (r2 = 0, r2 = 1, r2 = 2, just above 1) and random ones outside the
    unit disc, in turn"""
    fixed = [(d1, d2) for _, d1, d2, acc in polar_edges() if not acc]
    rs = np.random.RandomState(seed)
    d = rs.randint(0, 1 << 53, (2, 8 * n + 64), dtype=np.int64)
    _, _, _, acc = attempts(words_for(d[0], d[1]))
    d1, d2 = d[0][~acc][:n].copy(), d[1][~acc][:n].copy()
    for i in range(0, n, 7):
        d1[i], d2[i] = fixed[(i // 7) % len(fixed)]
    return d1, d2


def rejection_stream(accepted: int = 256, every: int = 1000, seed: int = 0):
    """(d1, d2): `accepted` blocks of every - 1 rejected attempts followed by one accepted attempt, so the last attempt needed is
    the stream's last"""
    a1, a2 = random_accepted(accepted, seed)
    r1, r2 = random_rejected(accepted * (every - 1), seed + 1)
    d1 = np.concatenate([r1.reshape(accepted, every - 1), a1[:, None]], axis=1).ravel()
    d2 = np.concatenate([r2.reshape(accepted, every - 1), a2[:, None]], axis=1).ravel()
    return d1, d2


def near_midpoint_attempts(n_cand: int = 2_000_000, keep: int = 20_000, seed: int = 2026):
    """(d1, d2) of accepted attempts whose log(r2) lies within 2^-6 ulp of a rounding midpoint: n_cand candidates with log-uniform
    |x1| = k 2^-52 (x2 = 0 in the first half, log-uniform in the second) are ranked by the long-double distance, and the `keep`
    closest distinct r2 kept where cr_log confirms the distance"""
    rs = np.random.RandomState(seed)
    k = np.floor(np.exp2(rs.uniform(0.0, 52.0, (2, n_cand)))).astype(np.int64)
    k[1, : n_cand // 2] = 0
    d = D_ZERO + k * (2 * rs.randint(0, 2, (2, n_cand)) - 1)
    _, _, r2, acc = attempts(words_for(d[0], d[1]))
    md = midpoint_distance(np.where(acc, r2, 0.5))
    md[~acc | np.isnan(md)] = 1.0
    _, first = np.unique(r2, return_index=True)
    first = first[md[first] < 1.0]
    sel = first[np.argsort(md[first], kind="stable")[:keep]]
    sel = np.sort(sel)
    _, dist = cr_logs(r2[sel])
    sel = sel[dist < 2.0 ** -6]
    return d[0][sel], d[1][sel]
