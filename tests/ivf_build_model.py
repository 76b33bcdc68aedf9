"""numpy model of the IVF build (kb2_build.cuh kmeans_train / assign_nearest / pq_encode_kernel, IvfIndex::train / add /
seal in kb2_index.cuh), as DESIGN §4.8 defines it.  Plain code of the definition, not a port of the kernels.

Random choices come from the C++ standard's std::mt19937_64:
  * k-means subsample: when n > 256 k, a partial Fisher-Yates shuffle of 0..n-1 (step i swaps i with i + rng() % (n - i))
    keeps the first 256 k positions, in that order;
  * init: the same partial shuffle of the nt training rows picks k rows, in order;
  * empty clusters, after each update, in ascending order ci: the populated cluster cj is found by scanning cj = 0, 1, ...
    (mod k) until (rng() >> 11) * 2^-53 < (count[cj] - 1) / (nt - k); then ci <- cj (1 +- 2^-10), cj <- cj (1 -+ 2^-10),
    '+' on ci's even coordinates, and count[ci] = count[cj] // 2, count[cj] -= count[ci].  Nothing is split when nt <= k;
  * IvfIndex::train seeds 1234 for the coarse quantizer and every PQ sub-quantizer, and 1234 + 7 for the PQ sample (the
    same partial shuffle, 65536 rows, when n > 65536).

Keys.  The device ranks lists by the norm-expanded key |x|^2 + |c|^2 - 2<x, c> (L2) or -<x, c> (IP), evaluated in fp32:
the two norms and the dot product are fp32 sums of d products each (relative error <= d u of the sum of their absolute
terms, u = 2^-24), and two more roundings combine them.  So the fp32 key is within

    B(x, c) = (d + 3) u S(x, c),    S = |x|^2 + |c|^2 + 2 sum_i |x_i c_i|  (L2),   S = sum_i |x_i c_i|  (IP)

of the exact key.  On the wgmma path each operand is split into hi = tf32(a) and lo = tf32(a - hi) and the products
hi*hi + hi*lo + lo*hi are summed: the dropped lo*lo and the rounding of lo are each <= 2^-22 |a b|, and the rounding of hi
is absorbed exactly by lo, so a product is off by at most 3 * 2^-22 < 2^-20 of |a b|.  That adds 2^-20 times the dot
product part of S: 2^-20 * 2 sum|x_i c_i| (L2) or 2^-20 sum|x_i c_i| (IP).  A choice l of row x is correct when

    K(x, c_l) <= min_j K(x, c_j) + B(x, c_l) + B(x, c_j*),    j* the exact argmin,

with K the exact key.  PQ codes are ranked by the direct sum over the sub-vector of (r_t - q_t)^2 with r = fp32(x - c)
the residual: r is off by u |r|, each difference by u (|r| + |r - q|), a square by 2u (|r| |r - q| + (r - q)^2), and the
fused multiply-add chain of dsub terms adds dsub u of the sum, so a code q is correct when its key is within
B_pq = (dsub + 3) u sum_t ((r_t - q_t)^2 + 2 |r_t| |r_t - q_t|) of the best code's, both bounds added as above.

On small-integer data (|values| <= 8) every key is an integer below 2^24 on both contractions (tf32 holds such values
whole and lo = 0), so the device must equal the exact argmin, first minimum on ties.

A centroid update is fp32(sum of the cluster's points) * fp32(1 / cnt); the device sums in its own fixed order, so a
coordinate is within (cnt + 1) u mean_p |x_pj| of the exact mean (exact on integer data, where the sum is exact)."""
import numpy as np

M64 = (1 << 64) - 1
U = 2.0 ** -24
TF32_TERM = 2.0 ** -20
KMEANS_NITER = 25
KMEANS_SEED = 1234
PQ_SAMPLE_SEED = 1234 + 7
PQ_SAMPLE_ROWS = 256 * 256
NLIST_MIN_ROWS = 39   # train() reduces nlist to max(1, n / 39) when nlist * 39 > n


# ------------------------------------------------------------------------------------------------------- generator
class MT19937_64:
    """std::mt19937_64 (C++ [rand.predef]: the 10000th output of a default-constructed engine is 9981545732273789042)"""
    N, M = 312, 156
    A = 0xB5026F5AA96619E9
    UPPER, LOWER = 0xFFFFFFFF80000000, 0x7FFFFFFF

    def __init__(self, seed=5489):
        mt = [seed & M64]
        for i in range(1, self.N):
            mt.append((6364136223846793005 * (mt[-1] ^ (mt[-1] >> 62)) + i) & M64)
        self.mt, self.i = mt, self.N

    def _twist(self):
        mt, N, M = self.mt, self.N, self.M
        for i in range(N):
            x = (mt[i] & self.UPPER) | (mt[(i + 1) % N] & self.LOWER)
            mt[i] = mt[(i + M) % N] ^ (x >> 1) ^ (self.A if x & 1 else 0)
        self.i = 0

    def __call__(self):
        if self.i >= self.N:
            self._twist()
        y = self.mt[self.i]
        self.i += 1
        y ^= (y >> 29) & 0x5555555555555555
        y ^= (y << 17) & 0x71D67FFFEDA60000
        y ^= (y << 37) & 0xFFF7EEE000000000
        y ^= y >> 43
        return y & M64


def partial_shuffle(n, count, rng):
    """the first `count` positions of the partial Fisher-Yates shuffle of 0..n-1 (step i swaps i and i + rng() % (n - i))"""
    perm = list(range(n))
    for i in range(count):
        j = i + rng() % (n - i)
        perm[i], perm[j] = perm[j], perm[i]
    return np.array(perm[:count], np.int64)


# ------------------------------------------------------------------------------------------------------- k-means
class KMeansDraws:
    """The random choices of one kmeans_train(n, k, seed) call, in the order the call makes them.
    sample: the training rows (None: all n, in order); init: positions in the training rows of the k initial centroids;
    split(counts): the (ci, cj) pairs of one iteration, from that iteration's counts (the rng state carries over)."""

    def __init__(self, n, k, seed=KMEANS_SEED):
        assert n >= k >= 1
        self.rng = MT19937_64(seed)
        self.sample = partial_shuffle(n, 256 * k, self.rng) if n > 256 * k else None
        self.nt = n if self.sample is None else 256 * k
        self.k = k
        self.init = partial_shuffle(self.nt, k, self.rng)

    def split(self, counts):
        hc = [int(c) for c in counts]
        k, nt = self.k, self.nt
        pairs = []
        for ci in range(k):
            if hc[ci] != 0:
                continue
            if nt <= k:
                break
            cj = 0
            while True:
                pr = (hc[cj] - 1.0) / float(nt - k)
                r = float(self.rng() >> 11) * (1.0 / 9007199254740992.0)
                if r < pr:
                    break
                cj = (cj + 1) % k
            pairs.append((ci, cj))
            hc[ci] = hc[cj] // 2
            hc[cj] -= hc[ci]
        return pairs


def apply_splits(C, pairs, tol=None):
    """the split pairs applied in order.  Without tol: to fp32 centroids C, as the device does (a copy is returned).
    With tol (per-coordinate error bound of C): to float64 centroids, returning (C, tol) with tol carried through the
    copies and widened by the device's fp32 rounding of the products."""
    up, dn = 1.0 + 2.0 ** -10, 1.0 - 2.0 ** -10
    if tol is None:
        C = np.array(C, np.float32, copy=True)
        up, dn = np.float32(up), np.float32(dn)
    else:
        C = np.array(C, np.float64, copy=True)
        T = np.array(tol, np.float64, copy=True)
    even = (np.arange(C.shape[1]) % 2) == 0
    for ci, cj in pairs:
        v = C[cj].copy()
        C[ci] = np.where(even, v * up, v * dn)
        C[cj] = np.where(even, v * dn, v * up)
        if tol is not None:
            T[ci] = T[cj] = T[cj] * up + 2.0 * U * np.abs(v)
    return C if tol is None else (C, T)


def lloyd_means(X, A, C_prev):
    """(C, mean, cnt, mabs): C the fp32 update fp32(sum x) * fp32(1 / cnt) over the points A == c (the device's value on
    integer data, where the sum is exact), mean the exact float64 mean, cnt the counts, mabs the mean |x| per coordinate.
    Empty clusters keep C_prev in C and mean."""
    X = np.asarray(X, np.float32)
    k = C_prev.shape[0]
    cnt = np.bincount(A, minlength=k)
    S = np.zeros(C_prev.shape, np.float64)
    Sa = np.zeros(C_prev.shape, np.float64)
    np.add.at(S, A, X.astype(np.float64))
    np.add.at(Sa, A, np.abs(X.astype(np.float64)))
    C = np.array(C_prev, np.float32, copy=True)
    mean = C.astype(np.float64)
    mabs = np.zeros(C_prev.shape, np.float64)
    nz = cnt > 0
    inv = np.float32(1.0) / cnt[nz].astype(np.float32)
    C[nz] = S[nz].astype(np.float32) * inv[:, None]
    mean[nz] = S[nz] / cnt[nz, None]
    mabs[nz] = Sa[nz] / cnt[nz, None]
    return C, mean, cnt, mabs


def mean_tolerance(cnt, mabs):
    """(cnt + 1) u mean|x|: how far a device centroid may lie from the exact mean of its cnt points"""
    return (np.asarray(cnt, np.float64)[:, None] + 1.0) * U * mabs


def check_means(C_got, want, cnt, mabs, exact=False, what=""):
    """every populated cluster's centroid within mean_tolerance of the exact mean `want` (bit for bit equal to the fp32
    update `want` when exact)"""
    nz = cnt > 0
    got, w = np.asarray(C_got, np.float32)[nz], np.asarray(want)[nz]
    if exact:
        bad = np.nonzero((got.view(np.uint32) != w.astype(np.float32).view(np.uint32)).any(1))[0]
    else:
        bad = np.nonzero((np.abs(got.astype(np.float64) - w) > mean_tolerance(cnt, mabs)[nz]).any(1))[0]
    if bad.size:
        c = np.nonzero(nz)[0][bad[0]]
        raise AssertionError(f"{what}: {bad.size} centroids are not the mean of their points, e.g. {c} "
                             f"(count {cnt[c]}): {got[bad[0]][:6]} vs {w[bad[0]][:6]}")


def match_nlist(nlist, n):
    return max(1, n // NLIST_MIN_ROWS) if nlist * NLIST_MIN_ROWS > n else nlist


# ------------------------------------------------------------------------------------------------------- keys
def uses_wgmma(n, d, k):
    """assign_nearest's contraction: the wgmma 3xTF32 kernel for k >= 512, d % 4 == 0 and a batch of n >= 1024 rows"""
    return k >= 512 and d % 4 == 0 and n >= 1024


def keys_and_bounds(X, C, metric, tf32):
    """(K, B) [n, k] float64: the exact norm-expanded key of every (row, centroid) and its fp32 error bound (docstring)"""
    X = np.asarray(X, np.float64)
    C = np.asarray(C, np.float64)
    d = X.shape[1]
    dot = X @ C.T
    ad = np.abs(X) @ np.abs(C).T
    if metric == "L2":
        xn, cn = (X * X).sum(1)[:, None], (C * C).sum(1)[None, :]
        K = xn + cn - 2.0 * dot
        S = xn + cn + 2.0 * ad
        B = (d + 3) * U * S + (TF32_TERM * 2.0 * ad if tf32 else 0.0)
    else:
        K = -dot
        B = (d + 3) * U * ad + (TF32_TERM * ad if tf32 else 0.0)
    return K, B


def _rows_per_chunk(k):
    return max(1, min(2048, (1 << 21) // max(k, 1)))


def exact_assign(X, C, metric):
    """argmin of the exact key, first minimum on ties (the device's result on small-integer data)"""
    out = np.empty(len(X), np.int64)
    step = _rows_per_chunk(len(C))
    for s in range(0, len(X), step):
        K, _ = keys_and_bounds(X[s:s + step], C, metric, False)
        out[s:s + step] = np.argmin(K, 1)
    return out


def check_assignment(X, C, A, metric, tf32, exact=False, what=""):
    """every row's list passes the rule of the docstring (equals the exact argmin, first minimum, when exact)"""
    A = np.asarray(A, np.int64)
    assert A.shape == (len(X),) and (A >= 0).all() and (A < len(C)).all(), f"{what}: list ids out of range"
    step = _rows_per_chunk(len(C))
    for s in range(0, len(X), step):
        K, B = keys_and_bounds(X[s:s + step], C, metric, tf32)
        a = A[s:s + step]
        r = np.arange(len(a))
        j = np.argmin(K, 1)
        if exact:
            bad = np.nonzero(a != j)[0]
        else:
            bad = np.nonzero(K[r, a] > K[r, j] + B[r, a] + B[r, j])[0]
        if bad.size:
            i = bad[0]
            raise AssertionError(f"{what}: {bad.size} rows in the wrong list, e.g. row {s + i} in {a[i]} (key "
                                 f"{K[i, a[i]]!r}, bound {B[i, a[i]]:.3g}), best {j[i]} (key {K[i, j[i]]!r}, "
                                 f"bound {B[i, j[i]]:.3g})")


# ------------------------------------------------------------------------------------------------------- PQ
def residuals(X, C, A):
    """fp32 residuals x - c_A (one fp32 subtraction per coordinate, as the device forms them)"""
    return np.asarray(X, np.float32) - np.asarray(C, np.float32)[np.asarray(A, np.int64)]


def pq_keys_and_bounds(R, pqc):
    """(K, B) [n, M, 256] float64: exact direct-difference key of each sub-vector residual against each codeword, and its
    fp32 error bound (docstring).  R: [n, M * dsub] fp32 residuals, pqc: [M, 256, dsub]."""
    M, ks, dsub = pqc.shape
    R = np.asarray(R, np.float64).reshape(len(R), M, 1, dsub)
    Q = np.asarray(pqc, np.float64)[None]
    df = R - Q
    K = (df * df).sum(-1)
    B = (dsub + 3) * U * (df * df + 2.0 * np.abs(R) * np.abs(df)).sum(-1)
    return K, B


def pq_encode(R, pqc):
    """the exact nearest codeword of every sub-vector, lowest code on ties"""
    out = np.empty((len(R), pqc.shape[0]), np.int64)
    for s in range(0, len(R), 1024):
        K, _ = pq_keys_and_bounds(R[s:s + 1024], pqc)
        out[s:s + 1024] = np.argmin(K, -1)
    return out


def check_codes(R, pqc, codes, exact=False, what=""):
    """every code passes the rule of the docstring (equals pq_encode when exact)"""
    codes = np.asarray(codes, np.int64)
    M = pqc.shape[0]
    assert codes.shape == (len(R), M), f"{what}: codes shape {codes.shape}"
    for s in range(0, len(R), 1024):
        K, B = pq_keys_and_bounds(R[s:s + 1024], pqc)
        c = codes[s:s + 1024]
        j = np.argmin(K, -1)
        kc = np.take_along_axis(K, c[..., None], -1)[..., 0]
        kj = np.take_along_axis(K, j[..., None], -1)[..., 0]
        bc = np.take_along_axis(B, c[..., None], -1)[..., 0]
        bj = np.take_along_axis(B, j[..., None], -1)[..., 0]
        bad = np.argwhere(c != j) if exact else np.argwhere(kc > kj + bc + bj)
        if len(bad):
            i, m = bad[0]
            raise AssertionError(f"{what}: {len(bad)} codes are not the nearest codeword, e.g. row {s + i} sub-quantizer "
                                 f"{m}: code {c[i, m]} (key {kc[i, m]!r}) vs {j[i, m]} (key {kj[i, m]!r})")


# ------------------------------------------------------------------------------------------------------- list layout
def layout(A, nlist):
    """rows of each list, stable-sorted by list: insertion order within a list"""
    A = np.asarray(A, np.int64)
    order = np.argsort(A, kind="stable")
    bounds = np.searchsorted(A[order], np.arange(nlist + 1))
    return [order[bounds[l]:bounds[l + 1]] for l in range(nlist)]


def check_layout(lists, labels, what=""):
    """lists: [nlist] arrays of exported labels.  Every label in exactly one list, in insertion order within a list.
    Returns the insertion position -> list assignment."""
    labels = np.asarray(labels, np.int64)
    pos_of = {int(v): i for i, v in enumerate(labels)}
    A = np.full(len(labels), -1, np.int64)
    for l, ids in enumerate(lists):
        p = np.array([pos_of.get(int(v), -1) for v in ids], np.int64)
        assert (p >= 0).all(), f"{what}: list {l} holds labels not added: {np.asarray(ids)[p < 0][:8]}"
        assert (A[p] == -1).all() and np.unique(p).size == p.size, f"{what}: list {l} repeats a row"
        assert (np.diff(p) > 0).all(), f"{what}: list {l} is not in insertion order: positions {p[:16]}"
        A[p] = l
    missing = np.nonzero(A < 0)[0]
    assert missing.size == 0, f"{what}: {missing.size} rows are in no list, e.g. label {labels[missing[0]]}"
    return A


def owner_table(counts, world):
    """list -> rank: lists by size, largest first (ties by list id), each onto the rank with the least rows so far
    (ties: the lowest rank)"""
    counts = np.asarray(counts, np.int64)
    owner = np.zeros(len(counts), np.int64)
    if world == 1:
        return owner
    load = [0] * world
    for l in np.argsort(-counts, kind="stable"):
        r = min(range(world), key=lambda q: (load[q], q))
        owner[l] = r
        load[r] += int(counts[l])
    return owner
