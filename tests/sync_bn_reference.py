"""numpy / Python-integer restatement of the synchronised batch norm's seven entry points (include/lidiff_b200.h, lb2_sync_bn_*).

Each function takes what its entry point takes and returns what it writes, as numpy arrays; the word arrays are int64 and combine
across ranks exactly as the kernels' do (`combine_max`, `combine_sum`).  fp64 element operations are numpy's, one rounding each; the
quotients of the integer sums are Python's int / int, which is correctly rounded.  Rows are processed in chunks so that millions of
rows need little memory."""
import math

import numpy as np

M32 = (1 << 32) - 1
CHUNK = 1 << 18


def _e(v):
    """e with |v| < 2^e (0 -> 0), per element"""
    return np.frexp(np.asarray(v, dtype=np.float64))[1].astype(np.int64)


def _chunks(n):
    for r0 in range(0, n, CHUNK):
        yield slice(r0, min(n, r0 + CHUNK))


def combine_max(words):
    return np.maximum.reduce([np.asarray(w) for w in words])


def combine_sum(words):
    return np.add.reduce([np.asarray(w) for w in words]).astype(np.int64)


def _split_sum(q):
    """(sum of q >> 32, sum of q & (2^32 - 1)) per column of the int64 array q"""
    return (q >> 32).sum(0, dtype=np.int64), (q & M32).sum(0, dtype=np.int64)


def _signed(hi, lo):
    return int(hi) * (1 << 32) + int(lo)


def _max_float(words):
    return np.asarray(words, dtype=np.int64).astype(np.uint32).view(np.float32).astype(np.float64)


def fwd_max(x):
    x = np.asarray(x, dtype=np.float32)
    n, c = x.shape
    w = np.zeros(2 * c, dtype=np.int64)
    for sl in _chunks(n):
        a = np.abs(x[sl])
        fin = np.isfinite(a)
        w[0::2] = np.maximum(w[0::2], np.where(fin, a, 0).astype(np.float32).view(np.uint32).max(0, initial=0))
        w[1::2] = np.maximum(w[1::2], (~fin).any(0))
    return w


def fwd_sum(x, max_words):
    x = np.asarray(x, dtype=np.float32)
    n, c = x.shape
    ok = max_words[1::2] == 0
    s = 62 - _e(_max_float(max_words[0::2]))
    w = np.zeros(2 * c + 1, dtype=np.int64)
    for sl in _chunks(n):
        q = np.rint(np.ldexp(x[sl][:, ok].astype(np.float64), s[ok])).astype(np.int64)
        hi, lo = _split_sum(q)
        w[0:2 * c:2][ok] += hi
        w[1:2 * c:2][ok] += lo
    w[2 * c] = n
    return w


def mean_of(max_words, sum_words):
    c = (len(sum_words) - 1) // 2
    n = int(sum_words[2 * c])
    mean = np.full(c, np.nan)
    for j in range(c):
        if max_words[2 * j + 1] == 0 and 0 < n < 1 << 31:
            s = 62 - int(_e(_max_float(max_words[2 * j])))
            mean[j] = math.ldexp(_signed(sum_words[2 * j], sum_words[2 * j + 1]) / n, -s)
    return mean


def _dev_shift(max_words, mean):
    return 62 - _e(_max_float(max_words[0::2]) + np.abs(mean))


def fwd_sumsq(x, max_words, sum_words):
    """(mean, sq_words)"""
    x = np.asarray(x, dtype=np.float32)
    n, c = x.shape
    mean = mean_of(max_words, sum_words)
    ok = max_words[1::2] == 0
    t = _dev_shift(max_words, mean)
    w = np.zeros(4 * c, dtype=np.int64)
    for sl in _chunks(n):
        d = x[sl][:, ok].astype(np.float64) - mean[ok]
        p = np.abs(np.rint(np.ldexp(d, t[ok])).astype(np.int64)).astype(np.uint64)
        # the canonical 32-bit limbs of p^2 (p < 2^63): p = a 2^32 + b
        a, b = p >> np.uint64(32), p & np.uint64(M32)
        bb, ab, aa = b * b, a * b, a * a
        l0 = bb & np.uint64(M32)
        t1 = (bb >> np.uint64(32)) + ((ab << np.uint64(1)) & np.uint64(M32))
        l1 = t1 & np.uint64(M32)
        t2 = (aa & np.uint64(M32)) + (ab >> np.uint64(31)) + (t1 >> np.uint64(32))
        l2 = t2 & np.uint64(M32)
        l3 = (aa >> np.uint64(32)) + (t2 >> np.uint64(32))
        for k, l in enumerate((l0, l1, l2, l3)):
            w[k::4][ok] += l.sum(0, dtype=np.uint64).astype(np.int64)
    return mean, w


def fwd_apply(x, max_words, sum_words, mean, sq_words, gamma, beta, eps, momentum, running_mean=None, running_var=None):
    """(var, invstd, y, running_mean', running_var') (the running pair None when not given)"""
    x = np.asarray(x, dtype=np.float32)
    c = x.shape[1]
    n = int(sum_words[2 * c])
    t = _dev_shift(max_words, mean)
    var = np.full(c, np.nan)
    for j in range(c):
        if max_words[2 * j + 1] == 0 and 0 < n < 1 << 31:
            T = sum(int(sq_words[4 * j + k]) << (32 * k) for k in range(4))
            var[j] = math.ldexp(T / n, -2 * int(t[j]))
    with np.errstate(invalid="ignore", divide="ignore"):
        invstd = 1.0 / np.sqrt(var + eps)
        g = np.ones(c) if gamma is None else np.asarray(gamma, dtype=np.float32).astype(np.float64)
        b = np.zeros(c) if beta is None else np.asarray(beta, dtype=np.float32).astype(np.float64)
        y = ((((x.astype(np.float64) - mean) * invstd) * g) + b).astype(np.float32)
        rm = rv = None
        if running_mean is not None:
            keep = 1.0 - momentum
            rm = ((keep * np.asarray(running_mean, np.float32).astype(np.float64)) + (momentum * mean)).astype(np.float32)
            unbiased = (var * float(n)) / float(n - 1) if n != 1 else np.full(c, np.nan)
            rv = ((keep * np.asarray(running_var, np.float32).astype(np.float64)) + (momentum * unbiased)).astype(np.float32)
    return var, invstd, y, rm, rv


def _g(dy, x, mean, invstd):
    with np.errstate(invalid="ignore", over="ignore"):
        return dy.astype(np.float64) * ((x.astype(np.float64) - mean) * invstd)


def bwd_max(dy, x, mean, invstd):
    dy, x = np.asarray(dy, np.float32), np.asarray(x, np.float32)
    n, c = x.shape
    w = np.zeros(3 * c, dtype=np.int64)
    for sl in _chunks(n):
        d, g = dy[sl], _g(dy[sl], x[sl], mean, invstd)
        fin = np.isfinite(d) & np.isfinite(g)
        w[0::3] = np.maximum(w[0::3], np.where(fin, np.abs(d), 0).astype(np.float32).view(np.uint32).max(0, initial=0))
        w[1::3] = np.maximum(w[1::3], np.where(fin, np.abs(g), 0).view(np.int64).max(0, initial=0))
        w[2::3] = np.maximum(w[2::3], (~fin).any(0))
    return w


def _bwd_shifts(max_words):
    sa = 62 - _e(_max_float(max_words[0::3]))
    sb = 62 - _e(np.asarray(max_words[1::3], dtype=np.int64).view(np.float64))
    return sa, sb


def bwd_sum(dy, x, mean, invstd, max_words):
    """(sum_words, dgamma, dbeta): the local words and this rank's parameter gradients"""
    dy, x = np.asarray(dy, np.float32), np.asarray(x, np.float32)
    n, c = x.shape
    ok = max_words[2::3] == 0
    sa, sb = _bwd_shifts(max_words)
    w = np.zeros(4 * c, dtype=np.int64)
    for sl in _chunks(n):
        d = dy[sl][:, ok]
        g = _g(d, x[sl][:, ok], mean[ok], invstd[ok])
        for k, (v, s) in enumerate(((d.astype(np.float64), sa), (g, sb))):
            hi, lo = _split_sum(np.rint(np.ldexp(v, s[ok])).astype(np.int64))
            w[2 * k::4][ok] += hi
            w[2 * k + 1::4][ok] += lo
    dgamma, dbeta = np.full(c, np.nan, np.float32), np.full(c, np.nan, np.float32)
    for j in np.nonzero(ok)[0]:
        dbeta[j] = np.float32(math.ldexp(float(_signed(w[4 * j], w[4 * j + 1])), -int(sa[j])))
        dgamma[j] = np.float32(math.ldexp(float(_signed(w[4 * j + 2], w[4 * j + 3])), -int(sb[j])))
    return w, dgamma, dbeta


def bwd_apply(dy, x, mean, invstd, gamma, max_words, sum_words, count):
    dy, x = np.asarray(dy, np.float32), np.asarray(x, np.float32)
    c = x.shape[1]
    n = int(count)
    sa, sb = _bwd_shifts(max_words)
    mdy, mg = np.full(c, np.nan), np.full(c, np.nan)
    for j in range(c):
        if max_words[3 * j + 2] == 0 and 0 < n < 1 << 31:
            mdy[j] = math.ldexp(_signed(sum_words[4 * j], sum_words[4 * j + 1]) / n, -int(sa[j]))
            mg[j] = math.ldexp(_signed(sum_words[4 * j + 2], sum_words[4 * j + 3]) / n, -int(sb[j]))
    g = np.ones(c) if gamma is None else np.asarray(gamma, np.float32).astype(np.float64)
    k = g * invstd
    with np.errstate(invalid="ignore", over="ignore"):
        xh = (x.astype(np.float64) - mean) * invstd
        return (k * ((dy.astype(np.float64) - mdy) - (xh * mg))).astype(np.float32)


def forward(xs, gamma, beta, eps=1e-5, momentum=0.1, running_mean=None, running_var=None):
    """the whole forward over the ranks' row blocks `xs`: dict of mean, var, invstd, ys (per rank), running_mean, running_var and the
    combined words"""
    mw = combine_max([fwd_max(x) for x in xs])
    sw = combine_sum([fwd_sum(x, mw) for x in xs])
    parts = [fwd_sumsq(x, mw, sw) for x in xs]
    mean = parts[0][0]
    qw = combine_sum([p[1] for p in parts])
    out = [fwd_apply(x, mw, sw, mean, qw, gamma, beta, eps, momentum, running_mean, running_var) for x in xs]
    var, invstd, _, rm, rv = out[0]
    return {"mean": mean, "var": var, "invstd": invstd, "ys": [o[2] for o in out], "running_mean": rm, "running_var": rv,
            "max_words": mw, "sum_words": sw, "sq_words": qw}


def backward(dys, xs, fwd, gamma):
    """the whole backward: dict of dxs (per rank), dgammas, dbetas (per rank, local sums)"""
    mean, invstd = fwd["mean"], fwd["invstd"]
    mw = combine_max([bwd_max(dy, x, mean, invstd) for dy, x in zip(dys, xs)])
    loc = [bwd_sum(dy, x, mean, invstd, mw) for dy, x in zip(dys, xs)]
    sw = combine_sum([l[0] for l in loc])
    n = fwd["sum_words"][-1]
    return {"dxs": [bwd_apply(dy, x, mean, invstd, gamma, mw, sw, n) for dy, x in zip(dys, xs)],
            "dgammas": [l[1] for l in loc], "dbetas": [l[2] for l in loc]}
