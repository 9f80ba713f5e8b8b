"""The two wgmma GEMM kernels of the MLPs vs torch.matmul on the same bf16 operands (fp32 accumulate):
`layer_gemm_kernel` (K-major operands, persistent, register accumulators) through dgl_gemm_bf16 and
`dw_gemm_kernel` (MN-major operands straight from the blocked activations) through dgl_gemm_tn_bf16."""
import ctypes

import pytest
import torch

import util

pytestmark = pytest.mark.gpu


def _ws(M, N, K):
    import _dgm_lib
    n = _dgm_lib.c_size_t()
    _dgm_lib.check(_dgm_lib.lib().dgl_gemm_ws_bytes(M, N, K, ctypes.byref(n)), "dgl_gemm_ws_bytes")
    return torch.empty(n.value, dtype=torch.uint8, device="cuda"), n.value


def run(M, N, K, bias=False, relu=False, lda=None, ldb=None):
    import _dgm_lib
    lib = _dgm_lib.lib()
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    lda, ldb = lda or K, ldb or K
    A = torch.zeros(M, lda).bfloat16().cuda()
    B = torch.zeros(N, ldb).bfloat16().cuda()
    A[:, :K] = torch.randn(M, K, generator=g).bfloat16().cuda()
    B[:, :K] = torch.randn(N, K, generator=g).bfloat16().cuda()
    b = torch.randn(N, generator=g).cuda() if bias else None
    ldc = (N + 3) // 4 * 4
    C = torch.zeros(M, ldc, device="cuda")
    ws, nbytes = _ws(M, N, K)
    rc = lib.dgl_gemm_bf16(M, N, K, A.data_ptr(), lda, B.data_ptr(), ldb, b.data_ptr() if bias else None,
                           int(relu), C.data_ptr(), ldc, ws.data_ptr(), nbytes, _dgm_lib.stream_ptr())
    _dgm_lib.check(rc, "dgl_gemm_bf16")
    ref = A[:, :K].float() @ B[:, :K].float().t()
    if bias:
        ref = ref + b
    if relu:
        ref = ref.clamp_min(0)
    return C[:, :N], ref


@pytest.mark.parametrize("M,N,K", [(128, 256, 256), (128, 32, 64), (300, 256, 96), (1000, 16, 256), (257, 96, 352),
                                   (4096, 256, 256), (128, 256, 16), (100_000, 256, 256), (50_000, 13, 256), (300, 256, 352),
                                   (777, 30, 250)])
def test_layer_gemm_matches_torch(M, N, K):
    C, ref = run(M, N, K)
    assert util.rel_err(C, ref) < 2e-5


def test_layer_gemm_epilogue_and_strides():
    C, ref = run(500, 256, 256, bias=True, relu=True, lda=264, ldb=272)
    assert util.rel_err(C, ref) < 2e-5
    C, ref = run(70_000, 48, 352, bias=True)
    assert util.rel_err(C, ref) < 2e-5


def run_tn(P, Mf, Nf, transpose=False):
    import _dgm_lib
    lib = _dgm_lib.lib()
    g = torch.Generator().manual_seed(P + 5 * Mf + 11 * Nf)
    X = torch.randn(P, Mf, generator=g).bfloat16().cuda()
    Y = torch.randn(P, Nf, generator=g).bfloat16().cuda()
    rows, cols = (Nf, Mf) if transpose else (Mf, Nf)
    ldc = (cols + 3) // 4 * 4
    C = torch.zeros(rows, ldc, device="cuda")
    ws, nbytes = _ws(P, 256, 256)
    rc = lib.dgl_gemm_tn_bf16(P, Mf, Nf, X.data_ptr(), Mf, Y.data_ptr(), Nf, C.data_ptr(), ldc, int(transpose),
                              ws.data_ptr(), nbytes, _dgm_lib.stream_ptr())
    _dgm_lib.check(rc, "dgl_gemm_tn_bf16")
    ref = X.float().t() @ Y.float()
    return C[:, :cols], (ref.t() if transpose else ref)


@pytest.mark.parametrize("P,Mf,Nf,tr", [(128, 256, 256, False), (1000, 256, 96, False), (5000, 256, 16, False),
                                        (4097, 256, 16, True), (3000, 256, 32, True), (100_000, 256, 256, False),
                                        (20_000, 200, 100, False)])
def test_dw_gemm_matches_torch(P, Mf, Nf, tr):
    C, ref = run_tn(P, Mf, Nf, tr)
    assert util.rel_err(C, ref) < 1e-4
