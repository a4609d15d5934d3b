"""GPU: tensor-core building blocks of the fused MLP (wgmma bf16x3 GEMM with A from registers) vs fp32/fp64 torch."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _lib():
    from tetranerf.utils.extension import tetranerf_cpp_extension as ext

    lib = ctypes.CDLL(ext.LIBRARY_PATH)
    lib.tn_last_error.restype = ctypes.c_char_p
    return lib


@pytest.mark.parametrize("K", [64, 128])
@pytest.mark.parametrize("scale", [1.0, 1e-4])
def test_debug_gemm_bf16x3(K, scale):
    lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(K)
    A = (torch.randn((128, K), generator=g) * scale).to(DEV)
    W = ((torch.rand((128, K), generator=g) * 2 - 1) / K**0.5).to(DEV)
    out = torch.full((128, 128), float("nan"), device=DEV)
    rc = lib.tn_debug_gemm_bf16x3(0, ctypes.c_void_p(A.data_ptr()), ctypes.c_void_p(W.data_ptr()), ctypes.c_uint32(K),
                                  ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(0))
    assert rc == 0, lib.tn_last_error()
    ref = (A.double() @ W.double().T)
    err = (out.double() - ref).abs().max().item()
    mag = ref.abs().max().item()
    print(f"K={K} scale={scale}: max abs err {err:.3e} (max |ref| {mag:.3e}, rel {err/mag:.3e})")
    assert err <= 2e-5 * mag, (err, mag)
    # a plain single-pass bf16 product would be ~1e-2 relative: make sure the lo terms are really in
    bf = (A.bfloat16().double() @ W.bfloat16().double().T - ref).abs().max().item()
    assert err < 0.05 * bf


def _gemm_modes(lib, mode, N, lbo, sbo, kstep, P, Q):
    out = torch.full((128, 128), float("nan"), device=DEV)
    rc = lib.tn_debug_gemm_modes(0, mode, ctypes.c_uint32(N), ctypes.c_uint32(lbo), ctypes.c_uint32(sbo), ctypes.c_uint32(kstep),
                                 ctypes.c_void_p(P.data_ptr()), ctypes.c_void_p(Q.data_ptr()), ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(0))
    assert rc == 0, lib.tn_last_error()
    torch.cuda.synchronize()
    return out[:, :N]


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("N", [128, 64])
def test_debug_gemm_operand_modes(mode, N):
    """the three operand forms of the fused MLP backward (K-major / MN-major shared-memory descriptors), bf16x3 accuracy"""
    lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(10 * mode + N)
    P = torch.randn((128, 128), generator=g).to(DEV)
    Q = (torch.randn((128, 128), generator=g) / 11.3).to(DEV)
    ref = {0: P.double() @ Q.double()[:N].T, 1: P.double() @ Q.double()[:, :N], 2: P.double().T @ Q.double()[:, :N]}[mode]
    out = _gemm_modes(lib, mode, N, 32768, 1024, 2048, P, Q)
    err = (out.double() - ref).abs().max().item()
    mag = ref.abs().max().item()
    print(f"mode={mode} N={N}: max abs err {err:.3e} (max |ref| {mag:.3e})")
    assert err <= 2e-5 * mag, (err, mag)
