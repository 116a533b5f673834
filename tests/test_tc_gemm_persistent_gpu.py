"""wgmma NT tiles with the GEMM self-test's plain store at shapes where every CTA runs many 64-row tiles per consumer
warpgroup: the persistent row loop, the wrap-around of the operand ring and the consumers' turn handoff, against an fp64
matmul on the device.  The last shape (K > 256) takes the variant that streams B through the ring.  The epilogue
functors at many tiles per CTA: test_nt_persistent_epilogue_gpu.py."""
import pytest

from test_tc_gemm_gpu import _run

pytestmark = pytest.mark.gpu

SHAPES = [(65536, 256, 256), (65613, 217, 256), (20000, 256, 320)]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_tc_gemm_split3_persistent(M, N, K):
    err = _run(M, N, K, 3)
    print(M, N, K, "split-3 rel-to-max err", err)
    assert err < 3e-5


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_tc_gemm_single_persistent(M, N, K):
    err = _run(M, N, K, 1)
    print(M, N, K, "single-bf16 rel-to-max err", err)
    assert err < 2e-2
