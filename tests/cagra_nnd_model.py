"""numpy model of GPU_CAGRA's NN-descent intermediate graph (build_algo NN_DESCENT), as defined in DESIGN §4.12 and at
cagra_nnd_join_kernel.  Keys, seeds and steps 2-5 are tests/cagra_model.py's.

On small-integer data every key is exact in fp32, so the device must reproduce this model bit for bit: G0, its keys, the
iteration count and updates(t)."""
import math

import numpy as np

from tests import cagra_model as cm

S_MAX = 32
DELTA = 1e-4   # stop when updates(t) <= DELTA * n * m
_BLOCK = 256   # joins applied per update (the update is a top-m of a totally ordered set: blocking does not change it)


def _splitmix64(z):
    """cagra_model.splitmix64 over a uint64 array"""
    with np.errstate(over="ignore"):
        z = (z + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def nnd_hash(src, tgt, t):
    """priority of source src among the reverse samples of target tgt at iteration t (smaller first, ties by src)"""
    src = np.asarray(src, np.uint64)
    tgt = np.asarray(tgt, np.uint64)
    return _splitmix64(np.uint64(cm.splitmix64(t)) ^ ((src << np.uint64(32)) | tgt)) >> np.uint64(32)


def init_ids(n, m):
    """L[i][j] = (i + 1 + (o_i + j * stride) mod (n - 1)) mod n, o_i = splitmix64(i) mod (n - 1), stride the first integer
    >= max(1, floor(0.618 (n - 1))) coprime to n - 1"""
    nm1 = n - 1
    stride = max(1, nm1 * 618 // 1000)
    while math.gcd(stride, nm1) != 1:
        stride += 1
    j = np.arange(m, dtype=np.int64)
    ids = np.empty((n, m), np.int64)
    for i in range(n):
        ids[i] = (i + 1 + (cm.splitmix64(i) % nm1 + j * stride) % nm1) % n
    return ids


def pair_keys(X, a, b, metric):
    """keys of the pairs (a[r], b[c]), [len(a), len(b)], -0 written as +0"""
    A = np.asarray(X[a], np.float64)
    B = np.asarray(X[b], np.float64)
    if metric == "L2":
        k = ((A[:, None, :] - B[None, :, :]) ** 2).sum(-1)
    else:
        k = -(A @ B.T)
    return k.astype(np.float32) + np.float32(0)


def _sort_rows(LK, LI, LF):
    o = np.lexsort((LI, LK))
    return (np.take_along_axis(LK, o, 1), np.take_along_axis(LI, o, 1), np.take_along_axis(LF, o, 1))


def _update(LK, LI, LF, tgt, key, vid):
    """L[u] <- the best m of L[u] u proposals(u) by (key, id), one entry per id; entering entries new.  A proposal worse
    than the current m-th key cannot enter."""
    m = LK.shape[1]
    keep = key <= LK[tgt, m - 1]
    tgt, key, vid = tgt[keep], key[keep], vid[keep]
    if not len(tgt):
        return
    rows = np.unique(tgt)
    U = np.concatenate([np.repeat(rows, m), tgt])
    K = np.concatenate([LK[rows].ravel(), key])
    V = np.concatenate([LI[rows].ravel(), vid])
    F = np.concatenate([LF[rows].ravel(), np.ones(len(tgt), bool)])
    E = np.concatenate([np.zeros(len(rows) * m, np.int8), np.ones(len(tgt), np.int8)])   # a present entry wins
    o = np.lexsort((E, V, U))
    U, K, V, F = U[o], K[o], V[o], F[o]
    first = np.ones(len(U), bool)
    first[1:] = (U[1:] != U[:-1]) | (V[1:] != V[:-1])
    U, K, V, F = U[first], K[first], V[first], F[first]
    o = np.lexsort((V, K, U))
    U, K, V, F = U[o], K[o], V[o], F[o]
    start = np.searchsorted(U, rows)
    pos = np.arange(len(U)) - np.repeat(start, np.diff(np.append(start, len(U))))
    sel = pos < m
    LK[rows] = K[sel].reshape(-1, m)
    LI[rows] = V[sel].reshape(-1, m)
    LF[rows] = F[sel].reshape(-1, m)


def nn_descent(X, m, niter, metric, history=False):
    """the NN-descent lists of the n rows of X: (ids [n, m], keys [n, m], iterations run, updates(t)); with history, also
    the (ids, keys, new flags) after each iteration"""
    X = np.asarray(X, np.float32)
    n = len(X)
    S = min(S_MAX, m)
    LI = init_ids(n, m)
    LK = np.stack([pair_keys(X, [i], LI[i], metric)[0] for i in range(n)])
    LF = np.ones((n, m), bool)
    LK, LI, LF = _sort_rows(LK, LI, LF)
    updates, hist = [], []
    for t in range(niter):
        # forward samples: the first <= S new entries (then old) and the first <= S old entries of each row
        sel_new = LF & (np.cumsum(LF, 1) <= S)
        sel_old = ~LF & (np.cumsum(~LF, 1) <= S)
        newf = [LI[i][sel_new[i]] for i in range(n)]
        oldf = [LI[i][sel_old[i]] for i in range(n)]
        LF &= ~sel_new
        # reverse samples: per target, the <= S sources of smallest (nnd_hash(src, tgt, t), src)
        rev = []
        for fw in (newf, oldf):
            src = np.repeat(np.arange(n), [len(f) for f in fw])
            tgt = np.concatenate(fw) if len(src) else np.zeros(0, np.int64)
            h = nnd_hash(src, tgt, t)
            o = np.lexsort((src, h, tgt))
            src, tgt = src[o], tgt[o]
            start = np.searchsorted(tgt, np.arange(n))
            end = np.searchsorted(tgt, np.arange(n), side="right")
            rev.append([src[start[i]:min(end[i], start[i] + S)] for i in range(n)])
        newr, oldr = rev
        # local joins, applied _BLOCK rows at a time
        for b0 in range(0, n, _BLOCK):
            tg, ky, vd = [], [], []
            for i in range(b0, min(n, b0 + _BLOCK)):
                cn = np.unique(np.concatenate([newf[i], newr[i]]))
                co = np.setdiff1d(np.concatenate([oldf[i], oldr[i]]), cn)
                C = np.concatenate([cn, co])
                if len(C) < 2:
                    continue
                isnew = np.arange(len(C)) < len(cn)
                K = pair_keys(X, C, C, metric)
                r, c = np.nonzero((isnew[:, None] | isnew[None, :]) & ~np.eye(len(C), dtype=bool))
                tg.append(C[r])
                ky.append(K[r, c])
                vd.append(C[c])
            if tg:
                _update(LK, LI, LF, np.concatenate(tg), np.concatenate(ky), np.concatenate(vd))
        upd = int(LF.sum())
        updates.append(upd)
        if history:
            hist.append((LI.copy(), LK.copy(), LF.copy()))
        if upd <= DELTA * n * m:
            break
    out = (LI, LK, len(updates), updates)
    return out + (hist,) if history else out


def build(X, igd, gd, metric, niter=20):
    """the graph of a build_algo NN_DESCENT build: steps 2-5 of cagra_model over the NN-descent G0"""
    n = len(X)
    m = min(igd, n - 1)
    g = min(gd, m)
    if g == 0:
        return np.full((n, 1), -1, np.int64)
    G0 = nn_descent(X, m, niter, metric)[0]
    P = cm.prune(G0, cm.detour_counts(G0), g)
    return cm.merge_rows(P, cm.reverse_lists(P, n))
