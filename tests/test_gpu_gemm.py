"""GPU parity: wgmma GEMM (csrc/gemm_tc.cu) vs an fp32 numpy product of the same fp16 operands, and vs the SIMT
cross-check kernel.  fp32 accumulation of exactly representable products: tolerance covers summation order only."""
import numpy as np
import pytest

from willow_inference_server_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def h():
    return _lib.Handle.frontend(0)


@pytest.mark.parametrize("M,N,K,bn", [
    (128, 128, 64, 128), (128, 256, 128, 256), (256, 384, 320, 128), (1536, 1280, 1280, 0),
    (384, 640, 3840, 256), (128, 51968, 128, 0), (2048, 5120, 1280, 256), (1536, 3840, 1280, 160), (256, 320, 192, 160),
])
def test_gemm_matches_fp32(h, M, N, K, bn):
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    a = rng.standard_normal((M, K), dtype=np.float32).astype(np.float16)
    w = rng.standard_normal((N, K), dtype=np.float32).astype(np.float16)
    c = h.debug_gemm(a, w, impl=0, bn=bn)
    if M * N * K <= 1536 * 1280 * 1280:
        ref = a.astype(np.float32) @ w.astype(np.float32).T
    else:  # sample rows to keep the CPU side quick
        rows = rng.choice(M, 64, replace=False)
        ref = a[rows].astype(np.float32) @ w.astype(np.float32).T
        c = c[rows]
    tol = 2e-5 * K ** 0.5 * 4 + 1e-4
    assert np.abs(c - ref).max() <= tol * max(1.0, np.abs(ref).max() / 10)


def test_gemm_structured_inputs_catch_layout_bugs(h):
    # A[m, k] = 1 if k == m % K else 0 -> C[m, n] = W[n, m % K]: any swizzle / descriptor slip permutes the result
    M, N, K = 256, 256, 192
    a = np.zeros((M, K), np.float16)
    a[np.arange(M), np.arange(M) % K] = 1
    w = (np.arange(N * K).reshape(N, K) % 1021).astype(np.float16)
    for bn in (128, 256):
        c = h.debug_gemm(a, w, impl=0, bn=bn)
        assert np.array_equal(c, w.astype(np.float32)[:, np.arange(M) % K].T)


def test_multicast_cluster_variant_is_bit_identical(h):
    # 2-CTA clusters with TMA-multicast W tiles vs the single-CTA kernel: same MMAs, same order -> identical bits
    rng = np.random.default_rng(3)
    for M, N, K, bn in [(256, 256, 128, 128), (512, 512, 640, 256), (1536, 3840, 1280, 256), (1536, 1280, 5120, 128),
                        (1536, 3840, 1280, 160)]:
        a = rng.standard_normal((M, K), dtype=np.float32).astype(np.float16)
        w = rng.standard_normal((N, K), dtype=np.float32).astype(np.float16)
        assert np.array_equal(h.debug_gemm(a, w, impl=0, bn=bn), h.debug_gemm(a, w, impl=0, bn=-bn))


def test_simt_crosscheck_agrees(h):
    rng = np.random.default_rng(1)
    a = rng.standard_normal((256, 256), dtype=np.float32).astype(np.float16)
    w = rng.standard_normal((384, 256), dtype=np.float32).astype(np.float16)
    assert np.abs(h.debug_gemm(a, w, impl=0) - h.debug_gemm(a, w, impl=1)).max() < 1e-3


def test_gemm_rejects_bad_shapes(h):
    with pytest.raises(ValueError):
        h.debug_gemm(np.zeros((100, 64), np.float16), np.zeros((128, 64), np.float16))
    with pytest.raises(ValueError):
        h.debug_gemm(np.zeros((128, 60), np.float16), np.zeros((128, 60), np.float16))


@pytest.mark.parametrize("R,N,K", [(5, 3840, 1280), (8, 1280, 5120), (1, 1280, 1280), (5, 5120, 1280), (3, 10240, 256), (5, 384, 384)])
def test_gemv_tc_matches_fp32_reference(h, R, N, K):
    # the wgmma skinny GEMV (weight rows on the MMA's M, activation rows on its N): x is rounded to fp16 inside, so the
    # reference multiplies the fp16-rounded x by the fp16 weights in fp32
    rng = np.random.default_rng(R * 1000 + N + K)
    x = rng.standard_normal((R, K)).astype(np.float32) * 3.0
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float16)
    bias = rng.standard_normal(N).astype(np.float32)
    got, _ = h.debug_gemv_tc(x, w, bias)
    want = x.astype(np.float16).astype(np.float32) @ w.astype(np.float32).T + bias
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 2e-3
    got2, _ = h.debug_gemv_tc(x, w, None)
    assert np.abs(got2 - (want - bias)).max() <= 2e-3
