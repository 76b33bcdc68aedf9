"""The wgmma (3xTF32, TMA-fed) contraction must reproduce the fp32 CUDA-core contraction, which in turn
is what the reference computes with src/simd fvec_L2sqr_ny / fvec_inner_products_ny (distances_ref.cc:22-38)."""
import ctypes

import numpy as np
import pytest

from knowhere_b200 import datagen

pytestmark = pytest.mark.gpu


def _keys(kb, torch, q, x, metric, use_tc):
    nq, d = q.shape
    nb = x.shape[0]
    ld = (nb + 3) & ~3
    out = torch.full((nq, ld), float("nan"), dtype=torch.float32, device="cuda")
    L = kb.lib()
    L.kb2_debug_gemm_keys.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                                      ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    kb._check(L.kb2_debug_gemm_keys(q.data_ptr(), nq, x.data_ptr(), nb, d, metric, use_tc, out.data_ptr(), 0))
    return out[:, :nb].cpu().numpy()


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("nq,nb,d", [(128, 128, 32), (100, 4096, 128), (333, 1003, 96), (1000, 5000, 768), (7, 130, 36)])
def test_tc_contraction_matches_fp32(kb, metric, nq, nb, d):
    torch = pytest.importorskip("torch")
    q = torch.from_numpy(datagen.uniform(nq, d, 1)).cuda()
    x = torch.from_numpy(datagen.uniform(nb, d, 2)).cuda()
    a = _keys(kb, torch, q, x, metric, 0)
    b = _keys(kb, torch, q, x, metric, 1)
    exact = (q.double() @ x.double().T).cpu().numpy()
    if metric == 0:
        exact = (q.double() ** 2).sum(1).cpu().numpy()[:, None] + (x.double() ** 2).sum(1).cpu().numpy()[None] - 2 * exact
    else:
        exact = -exact
    scale = float(np.abs(q.cpu().numpy()).max() * np.abs(x.cpu().numpy()).max() * d)
    err_fp32 = np.abs(a - exact).max() / scale
    err_tc = np.abs(b - exact).max() / scale
    print(f"nq={nq} nb={nb} d={d} metric={metric}: max err / scale  fp32 {err_fp32:.2e}  tc {err_tc:.2e}")
    assert not np.isnan(b).any()
    # fp32 FMA chain: ~1e-6; 3xTF32 (hi*hi + hi*lo + lo*hi, lo*lo dropped): a few 1e-6 at d=768.  Both far below
    # the spacing of candidate keys, and the k+16 best candidates are re-ranked exactly (finalize_kernel).
    assert err_tc < 6e-6 and err_fp32 < 2e-6
