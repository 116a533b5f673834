"""wgmma weight-gradient (TN) tiles against fp64 at the training step's shapes (P = 65 536 points, the benchmark's split
sizing; every tile width BN = 64 / 128 / 256 with its own ring depth) and the split-K flush with 8-byte reductions (C and
ldc 8-byte aligned) and with scalar ones (C off 8 bytes, or odd ldc)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _run_tn(P, N1, N2, nprod, c_off=0, seed=0):
    """C[N1][N2] (ldc = N2) starts c_off floats into its buffer; returns the errors of C and of the fused column sum,
    relative to their largest reference entry."""
    from avatarclip_b200 import _lib
    L = _lib.lib()
    L.avc_tc_gemm_tn_test.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.avc_tc_gemm_tn_test.restype = C.c_int
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(P, N1, generator=g).cuda()
    B = (torch.randn(P, N2, generator=g) * 0.1).cuda()
    buf = torch.randn(N1 * N2 + c_off, generator=g).cuda()
    base = buf[c_off:].clone().view(N1, N2)
    r8 = lambda n: (n + 7) // 8 * 8
    ws = torch.empty(4 * P * (r8(N1) + r8(N2)) + 8192, dtype=torch.uint8, device="cuda")
    cs = torch.ones(N1, device="cuda")
    _lib.check(L.avc_tc_gemm_tn_test(A.data_ptr(), B.data_ptr(), P, N1, N2, nprod, buf.data_ptr() + 4 * c_off,
                                     cs.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "avc_tc_gemm_tn_test")
    torch.cuda.synchronize()
    ref = base.double() + A.double().t() @ B.double()
    cref = 1.0 + A.double().sum(0)
    cerr = (cs.double() - cref).abs().max().item() / cref.abs().max().item()
    err = (buf[c_off:].view(N1, N2).double() - ref).abs().max().item() / ref.abs().max().item()
    return err, cerr


@pytest.mark.parametrize("P,N1,N2,c_off", [(65536, 256, 256, 0), (65536, 256, 39, 0), (65536, 217, 256, 0),
                                           (65536, 256, 256, 1), (70000, 200, 100, 0), (4096, 384, 64, 1)])
def test_tn_split3_step_shapes(P, N1, N2, c_off):
    err, cerr = _run_tn(P, N1, N2, 3, c_off)
    print(P, N1, N2, c_off, "TN split-3 rel-to-max err", err, "column sum", cerr)
    assert err < 3e-5
    assert cerr < 3e-5


@pytest.mark.parametrize("P,N1,N2", [(65536, 256, 256), (65536, 256, 39)])
def test_tn_single_step_shapes(P, N1, N2):
    err, cerr = _run_tn(P, N1, N2, 1)
    print(P, N1, N2, "TN single-bf16 rel-to-max err", err, "column sum", cerr)
    assert err < 2e-2
    assert cerr < 2e-2
