"""CPU checks of the MUVERA numpy model (tests/muvera_model.py) that the GPU tests hold the library to."""
import shutil

import numpy as np
import pytest

from tests import muvera_model as mm

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="g++ builds the projection generator")


def test_projections_are_drawn_per_repeat_from_seed_plus_r():
    P, R, d, S = 3, 4, 20, 42
    pr = mm.projections(P, R, d, S)
    assert pr.shape == (R, P, d) and pr.dtype == np.float32
    for r in range(R):
        assert np.array_equal(pr[r], mm.projections(P, 1, d, S + r)[0])
    # row-major P x d per repeat: the first P * d draws of the generator, in order
    assert np.array_equal(mm.projections(1, 1, P * d, S)[0, 0], pr[0].ravel())
    assert not np.array_equal(pr, mm.projections(P, R, d, S + 1))
    # int32 seeds wrap as the reference's int32 seed + r does in the generator's 32-bit seed
    assert np.array_equal(mm.projections(2, 2, 8, 2 ** 31 - 1)[1], mm.projections(2, 1, 8, -2 ** 31)[0])
    big = mm.projections(4, 8, 128, 7)
    assert abs(float(big.mean())) < 0.05 and abs(float(big.std()) - 1.0) < 0.05


def test_buckets_flip_with_the_sign_of_the_token():
    rng = np.random.default_rng(1)
    proj = mm.projections(5, 3, 16, 3)
    x = rng.standard_normal((200, 16)).astype(np.float32)
    b, amb = mm.buckets(x, proj)
    bn, ambn = mm.buckets(-x, proj)
    assert not amb.any() and not ambn.any()
    assert np.array_equal(bn, 31 - b)
    # a token on a hyperplane is ambiguous; the zero token is in the last bucket (every dot is >= 0)
    z, az = mm.buckets(np.zeros((1, 16), np.float32), proj)
    assert az.all() and (z == 31).all()


def test_fde_sums_in_token_order_and_means_by_count():
    rng = np.random.default_rng(2)
    P, R, d = 2, 3, 8
    proj = mm.projections(P, R, d, 9)
    lens = [0, 1, 5, 12]
    lims = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    x = rng.standard_normal((int(lims[-1]), d)).astype(np.float32)
    bkt, _ = mm.buckets(x, proj)
    s = mm.fde(x, lims, bkt, R, P, mean=False).reshape(len(lens), R, 1 << P, d)
    m = mm.fde(x, lims, bkt, R, P, mean=True).reshape(len(lens), R, 1 << P, d)
    assert not s[0].any() and not m[0].any()   # an empty document stays zero
    for i in range(1, len(lens)):
        for r in range(R):
            for b in range(1 << P):
                rows = x[lims[i]:lims[i + 1]][bkt[lims[i]:lims[i + 1], r] == b]
                acc = np.zeros(d, np.float32)
                for t in rows:
                    acc = acc + t
                assert np.array_equal(s[i, r, b], acc)
                want = acc * (np.float32(1) / np.float32(len(rows))) if len(rows) > 1 else acc
                assert np.array_equal(m[i, r, b], want)
    # one token: the token itself in its bucket of every repeat, mean or not
    assert np.array_equal(s[1], m[1])
    for r in range(R):
        assert np.array_equal(s[1, r, bkt[0, r]], x[0])


def test_ann_k():
    assert mm.ann_k(10, 3.0, 1000) == 30
    assert mm.ann_k(10, 3.0, 20) == 20
    assert mm.ann_k(1, 0.35, 50) == 1
    assert mm.ann_k(7, 0.35, 50) == 2
