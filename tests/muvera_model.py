"""A numpy restatement of the MUVERA strategy (DESIGN §4.11), the reference's emb_list_strategy_muvera.cc.

Projections.  Repeat r has a P x d matrix whose entries are drawn in order from std::normal_distribution<float>(0, 1) over
std::mt19937(S + r).  numpy has no such generator, so `projections` compiles a small C++ program that uses only <random>
(g++, the same standard library the reference links) and reads its output.

Buckets.  Token x falls in bucket sum of 2^p over the projections p with dot(proj_p, x) >= 0.  The model takes the dots in
float64.  The device adds the fp32 products in another order, so its dot can differ from the exact one by at most
gamma_d * sum |p_i x_i|, with gamma_d = d u / (1 - d u) and u = 2^-24 (any order of d fp32 fused multiply-adds, the
products included: Higham, Accuracy and Stability of Numerical Algorithms, §3.1).  A token whose float64 dot lies within
that bound of 0 for some projection is ambiguous: its bucket is not determined by the definition alone.

FDE.  Per (repeat, bucket) the tokens in the bucket are added in fp32, in token order, starting from 0 (the reference's
fvec_madd with factor 1.0f is one exact-rounded add per element); documents then scale each bucket holding c > 1 tokens
by float32(1 / c).
"""
import os
import subprocess
import tempfile

import numpy as np

U = 2.0 ** -24

_HELPER = r"""
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <random>
int main(int argc, char** argv) {
    const int P = atoi(argv[1]), R = atoi(argv[2]), d = atoi(argv[3]);
    const long long S = atoll(argv[4]);
    for (int r = 0; r < R; r++) {
        std::mt19937 rng((uint32_t)(S + r));
        std::normal_distribution<float> nd(0.0f, 1.0f);
        for (int i = 0; i < P * d; i++) {
            const float v = nd(rng);
            fwrite(&v, 4, 1, stdout);
        }
    }
    return 0;
}
"""
_EXE = None


def helper_exe():
    """path of the compiled projection generator (built once per process)"""
    global _EXE
    if _EXE is None:
        tmp = tempfile.mkdtemp(prefix="muvera_model_")
        src = os.path.join(tmp, "proj.cc")
        with open(src, "w") as f:
            f.write(_HELPER)
        exe = os.path.join(tmp, "proj")
        subprocess.run(["g++", "-std=c++17", "-O2", src, "-o", exe], check=True)
        _EXE = exe
    return _EXE


def projections(P, R, d, S):
    """[R, P, d] float32"""
    out = subprocess.run([helper_exe(), str(P), str(R), str(d), str(S)], capture_output=True, check=True).stdout
    return np.frombuffer(out, np.float32).reshape(R, P, d).copy()


def buckets(x, proj):
    """(bucket [n, R] int, ambiguous [n] bool) of float32 tokens x [n, d] under proj [R, P, d]"""
    R, P, d = proj.shape
    x64 = x.astype(np.float64)
    p64 = proj.astype(np.float64)
    dots = np.einsum("nd,rpd->nrp", x64, p64)
    mag = np.einsum("nd,rpd->nrp", np.abs(x64), np.abs(p64))
    gamma = d * U / (1 - d * U)
    amb = (np.abs(dots) <= gamma * mag).any(axis=(1, 2))
    bits = (dots >= 0).astype(np.int64) << np.arange(P)[None, None, :]
    return bits.sum(-1), amb


def fde(x, lims, bkt, R, P, mean):
    """encodings [n_items, R * 2^P * d] float32 of the items lims[i] .. lims[i + 1] of x, given their tokens' buckets"""
    B, d = 1 << P, x.shape[1]
    n_items = len(lims) - 1
    out = np.zeros((n_items, R, B, d), np.float32)
    for i in range(n_items):
        for r in range(R):
            cnt = np.zeros(B, np.int64)
            for t in range(lims[i], lims[i + 1]):
                b = bkt[t, r]
                out[i, r, b] = out[i, r, b] + x[t]   # fp32 add, token order
                cnt[b] += 1
            if mean:
                for b in range(B):
                    if cnt[b] > 1:
                        out[i, r, b] *= np.float32(1.0) / np.float32(cnt[b])
    return out.reshape(n_items, -1)


def encode(x, lims, proj, mean):
    """(encodings, ambiguous tokens) of the items of x under proj"""
    R, P, _ = proj.shape
    bkt, amb = buckets(x, proj)
    return fde(x, lims, bkt, R, P, mean), amb


def ann_k(k, ratio, n_docs):
    """min(max(int32(fp32(k) * fp32(ratio)), 1), n_docs)"""
    return int(min(max(int(np.float32(k) * np.float32(ratio)), 1), n_docs))
