"""Hardware self-test of the wgmma / TMA SW128 plumbing (csrc/wgmma.cuh) that the tensor-core correlation path is
built on: bf16 GEMMs through libfn2b200_test.so (csrc_test/fn2b200_test.h, csrc_test/wgmma_selftest.cu)."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("K", [64, 256])
def test_umma_gemm_matches_cpu(K):
    import testlib
    LIB = testlib.load()
    g = torch.Generator().manual_seed(K)
    A = torch.randn(128, K, generator=g).bfloat16()
    B = torch.randn(144, K, generator=g).bfloat16()
    Ad, Bd = A.cuda(), B.cuda()
    D = torch.full((128, 144), float("nan"), device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    testlib.check(LIB, LIB.fn2b200_test_wgmma_gemm_ss(ctypes.c_void_p(Ad.data_ptr()), ctypes.c_void_p(Bd.data_ptr()),
                                                     ctypes.c_void_p(D.data_ptr()), K, st), "test_wgmma_gemm_ss")
    torch.cuda.synchronize()
    ref = A.double() @ B.double().t()
    err = (D.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-5, err


@pytest.mark.parametrize("a_sw32", [0, 1])
def test_umma_gemm_noswizzle_a_mnmajor_b(a_sw32):
    """A built by threads (K-major, no swizzle or 32-byte swizzle), B^T = [K][N] row-major consumed as an MN-major
    SW128 operand -- the tensor-core backward's B form."""
    import testlib
    LIB = testlib.load()
    g = torch.Generator().manual_seed(7)
    A = torch.randn(128, 144, generator=g).bfloat16()
    Bt = torch.randn(144, 64, generator=g).bfloat16()
    Ad, Bd = A.cuda(), Bt.cuda()
    D = torch.full((128, 64), float("nan"), device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    testlib.check(LIB, LIB.fn2b200_test_wgmma_gemm_mn(ctypes.c_void_p(Ad.data_ptr()), ctypes.c_void_p(Bd.data_ptr()),
                                                     ctypes.c_void_p(D.data_ptr()), a_sw32, st), "test_wgmma_gemm_mn")
    torch.cuda.synchronize()
    ref = A.double() @ Bt.double()
    err = (D.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-5, err


@pytest.mark.parametrize("K", [64, 256])
def test_umma_gemm_a_from_tensor_memory(K):
    """A not from shared memory: Hopper's wgmma takes A from registers (fragment = rows lane/4 (+8), k pairs 2 (lane%4)
    (+8)), here loaded straight from global memory; B from shared memory (K-major SW128, TMA)."""
    import testlib
    LIB = testlib.load()
    g = torch.Generator().manual_seed(100 + K)
    A = torch.randn(128, K, generator=g).bfloat16()
    B = torch.randn(144, K, generator=g).bfloat16()
    Ad, Bd = A.cuda(), B.cuda()
    D = torch.full((128, 144), float("nan"), device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    testlib.check(LIB, LIB.fn2b200_test_wgmma_gemm_rs(ctypes.c_void_p(Ad.data_ptr()), ctypes.c_void_p(Bd.data_ptr()),
                                                     ctypes.c_void_p(D.data_ptr()), K, st), "test_wgmma_gemm_rs")
    torch.cuda.synchronize()
    ref = A.double() @ B.double().t()
    err = (D.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-5, err


@pytest.mark.parametrize("K", [64, 256])
def test_umma_gemm_a_copied_to_tensor_memory_by_tcgen05_cp(K):
    """A staged by TMA into a 128-byte-swizzled shared-memory tile (the forward's A layout) and read from there into the
    wgmma register fragments (the name is the one this check had when A went to Blackwell's tensor memory)."""
    import testlib
    LIB = testlib.load()
    g = torch.Generator().manual_seed(200 + K)
    A = torch.randn(128, K, generator=g).bfloat16()
    B = torch.randn(144, K, generator=g).bfloat16()
    Ad, Bd = A.cuda(), B.cuda()
    D = torch.full((128, 144), float("nan"), device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    testlib.check(LIB, LIB.fn2b200_test_wgmma_gemm_rs_tma(ctypes.c_void_p(Ad.data_ptr()), ctypes.c_void_p(Bd.data_ptr()),
                                                       ctypes.c_void_p(D.data_ptr()), K, st), "test_wgmma_gemm_rs_tma")
    torch.cuda.synchronize()
    ref = A.double() @ B.double().t()
    err = (D.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-5, err
