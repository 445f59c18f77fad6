"""GPU: the training path's wgmma GEMM in isolation (csrc/nb_train.cu::gemm_tf32x3_kernel) against fp64 matmuls:
both operand layouts, ragged M / K, N tiles, bias + relu + mask epilogues, split reductions with atomics, and the range of
magnitudes gradients have (fp16 pairs would underflow there)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def run(M, N, K, a_kc, b_kc, splits=1, bias=False, relu=False, mask=False, scale_a=1.0, scale_b=1.0, seed=0):
    from neuralbody_b200 import capi
    lib = capi.load()
    g = torch.Generator().manual_seed(seed)
    A = torch.randn((M, K), generator=g) * scale_a
    B = torch.randn((N, K), generator=g) * scale_b
    dev = "cuda:0"
    a_d = (A if a_kc else A.t().contiguous()).to(dev)
    b_d = (B if b_kc else B.t().contiguous()).to(dev)
    bias_t = torch.randn((N,), generator=g) if bias else None
    mask_t = torch.randn((M, N), generator=g) if mask else None
    c = torch.zeros((M, N), dtype=torch.float32, device=dev)
    bd = bias_t.to(dev) if bias else None
    md = mask_t.to(dev) if mask else None
    st = lib.nb_debug_gemm_tf32x3(a_d.data_ptr(), b_d.data_ptr(), c.data_ptr(), M, N, K, int(a_kc), int(b_kc), splits,
                                  bd.data_ptr() if bias else None, int(relu), md.data_ptr() if mask else None,
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream))
    capi.check(st, "nb_debug_gemm_tf32x3")
    torch.cuda.synchronize()
    ref = A.double() @ B.double().t()
    if bias:
        ref = ref + bias_t.double()
    if relu:
        ref = torch.relu(ref)
    if mask:
        ref = torch.where(mask_t > 0, ref, torch.zeros_like(ref))
    got = c.cpu().double()
    scale = float((A.double().abs() @ B.double().abs().t()).max())      # the magnitude the rounding errors scale with
    return float((got - ref).abs().max()) / scale, float(ref.abs().max())


@pytest.mark.parametrize("a_kc,b_kc", [(1, 1), (1, 0), (0, 0), (0, 1)])
def test_layouts(a_kc, b_kc):
    err, mx = run(300, 256, 352, a_kc, b_kc)
    print("layouts a_kc=%d b_kc=%d: rel err %.3e (|ref| max %.1f)" % (a_kc, b_kc, err, mx))
    assert err < 2e-6


def test_forward_layer_epilogue():
    err, _ = run(1000, 256, 352, 1, 0, bias=True, relu=True)
    assert err < 2e-6
    err, _ = run(517, 144, 352, 1, 1, bias=True)
    assert err < 2e-6


def test_dgrad_mask_and_n_tiles():
    err, _ = run(700, 352, 256, 1, 0, mask=True)          # two N tiles (256 + 96)
    assert err < 2e-6
    err, _ = run(260, 256, 144, 1, 0, mask=True)          # K = 144: a ragged last chunk
    assert err < 2e-6


def test_wgrad_split_reduction():
    err, _ = run(256, 352, 10007, 0, 0, splits=36)        # reduction over a ragged list, fp32 atomics
    assert err < 2e-6
    err, _ = run(144, 352, 4099, 0, 0, splits=72)         # M = 144: second row tile has 16 live rows
    assert err < 2e-6


def test_gradient_magnitudes():
    err, mx = run(256, 256, 256, 1, 0, scale_a=1e-7, scale_b=1.0)
    print("tiny operands: rel err %.3e, |ref| max %.3e" % (err, mx))
    assert err < 2e-6 and mx > 0
