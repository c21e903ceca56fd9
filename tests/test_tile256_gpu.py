"""The 128 x 256 GEMM tile (gemm_wgmma.cu, gemm_kernel<256>: wgmma m64n256k16, 4-stage ring, consumers at 232 registers)
at its edges, with the exact-integer method and the guard bands of tests/test_hopper_kernels_gpu.py, and the three-way
tile-width rule of the dispatcher.  Every edge shape runs twice: with the width the dispatcher picks and forced to 256."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_hopper_kernels_gpu as H  # noqa: E402
from test_hopper_kernels_gpu import (ACT_GELU, ACT_GELU_TANH, ACT_NONE, ACT_RELU, ACT_SILU, ACT_SWIGLU,  # noqa: E402
                                     assert_exact, assert_guard, assert_within, elementwise_bound, gemm_ref, guarded,
                                     small_ints)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from internnav_b200 import _lib
    _lib.lib()
    return _lib


def tile_width(M, N, K, sms):
    """The dispatcher's rule (gemm_wgmma.cu, gemm_bf16): least waves x (BN + 48), ties to the wider tile; 256 is a candidate
    only for a W of more than 32 MB."""
    tm = (M + 127) // 128

    def cost(bn):
        return (tm * ((N + bn - 1) // bn) + sms - 1) // sms * (bn + 48)
    bn = 128 if cost(128) <= cost(64) else 64
    if N * K * 2 > (32 << 20) and cost(256) <= cost(bn):
        bn = 256
    return bn


# N % 256 in {8, 136, 248}, M % 128 in {1, 127}, K = 8 and K % 64 = 56; SM + 1 and 2 SM + 1 tiles of width 256 with 5 and 6
# k-blocks per tile, so the 4-stage ring's slot and phase differ at every tile start inside a CTA; and a W of over 32 MB,
# which the dispatcher gives the 256-wide tile and a raster group of 18 M tiles (20 M tiles: the last group is short).
SHAPES = [
    ("n8_m1_k8only", lambda s: (129, 264, 8)),
    ("n136_m127_k56", lambda s: (255, 392, 120)),
    ("n248_m1_k56", lambda s: (257, 504, 184)),
    ("tiles_sm_plus_1", lambda s: (s * 128 + 1, 256, 312)),
    ("tiles_2sm_plus_1", lambda s: (2 * s * 128 + 127, 256, 376)),
    ("w_over_32mb_n136_k8", lambda s: (2500, 4744, 3592)),
]


def test_shape_set_reaches_every_tile_width():
    sms = H._sms()
    picked = {name: tile_width(*f(sms), sms) for name, f in SHAPES}
    assert set(picked.values()) == {64, 128, 256}, picked
    assert picked["w_over_32mb_n136_k8"] == 256
    for name, want in (("tiles_sm_plus_1", sms + 1), ("tiles_2sm_plus_1", 2 * sms + 1)):
        M, N, _ = dict(SHAPES)[name](sms)
        assert ((M + 127) // 128) * ((N + 255) // 256) == want


@pytest.mark.parametrize("tile_n", [0, 256], ids=["dispatched", "forced256"])
@pytest.mark.parametrize("name,shape", SHAPES, ids=[n for n, _ in SHAPES])
def test_exact_shapes(L, name, shape, tile_n):
    M, N, K = shape(H._sms())
    gen = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = small_ints((M, K), -2, 2, gen, device="cuda")
    w = small_ints((N, K), -2, 2, gen, device="cuda")
    bias = small_ints((N,), -8, 8, gen, torch.float32, "cuda")
    gamma = small_ints((N,), -2, 2, gen, torch.float32, "cuda")
    res = small_ints((M, N), -64, 64, gen, device="cuda")
    ref, _ = gemm_ref(a, w, bias, gamma, res)
    outs = []
    for _ in range(2):
        buf, out = guarded(M, N, torch.bfloat16, "cuda")
        L.gemm_tile(a, w, out, bias, gamma, res, tile_n=tile_n)
        torch.cuda.synchronize()
        assert_guard(buf, out, name)
        outs.append(out.clone())
    assert_exact(outs[0], ref, "%s M=%d N=%d K=%d tile %d" % (name, M, N, K, tile_n))
    assert torch.equal(outs[0], outs[1]), "second call differs"


@pytest.mark.parametrize("store", ["tma", "fp32", "direct"])
@pytest.mark.parametrize("act", [ACT_NONE, ACT_GELU, ACT_RELU, ACT_SWIGLU, ACT_GELU_TANH, ACT_SILU])
def test_epilogues_forced_256(L, act, store):
    """Every activation with no epilogue operand and with bias + gamma + residual (SwiGLU: bias only), through the TMA-store
    path, the fp32 path and the register-store path of a misaligned bf16 view.  N % 256 = 144, M % 128 = 127, K % 64 = 56."""
    if act == ACT_SWIGLU and store == "fp32":
        pytest.skip("the SwiGLU epilogue writes bf16")
    M, N, K = 255, 400, 120
    gen = torch.Generator().manual_seed(act * 10 + len(store))
    a = small_ints((M, K), -2, 2, gen, device="cuda")
    w = small_ints((N, K), -1, 1, gen, device="cuda")
    n_out = N // 2 if act == ACT_SWIGLU else N
    bias = small_ints((N,), -6, 6, gen, torch.float32, "cuda")
    gamma = small_ints((n_out,), -2, 2, gen, torch.float32, "cuda")
    res = small_ints((M, n_out), -32, 32, gen, device="cuda")
    dtype = torch.float32 if store == "fp32" else torch.bfloat16
    for epi in ((None, None, None), (bias, None, None) if act == ACT_SWIGLU else (bias, gamma, res)):
        left, right = (4, 4) if store == "direct" else (8, 8)
        buf, out = guarded(M, n_out, dtype, "cuda", left=left, right=right)
        assert (out.data_ptr() % 16 != 0) == (store == "direct")
        L.gemm_tile(a, w, out, *epi, act=act, tile_n=256)
        torch.cuda.synchronize()
        what = "act=%d %s %s" % (act, store, "full" if epi[0] is not None else "none")
        assert_guard(buf, out, what)
        ref, mag = gemm_ref(a, w, *epi, act=act)
        if act in (ACT_NONE, ACT_RELU):
            assert_exact(out, ref, what)
        else:
            assert_within(out, ref, elementwise_bound(ref, mag, K, bf16_out=dtype == torch.bfloat16), what)


@pytest.mark.parametrize("tile_n", [128, 256])
def test_row_add_and_row_remap(L, tile_n):
    """The patch-embedding epilogue: out[(r / P) * (P + 1) + r % P + 1] = A W^T + bias + row_add[r % P]; row 0 of every
    group of P + 1 output rows (the class token's) is not written."""
    P, groups, N, K = 51, 5, 392, 56
    M = P * groups
    gen = torch.Generator().manual_seed(tile_n)
    a = small_ints((M, K), -2, 2, gen, device="cuda")
    w = small_ints((N, K), -2, 2, gen, device="cuda")
    bias = small_ints((N,), -8, 8, gen, torch.float32, "cuda")
    row_add = small_ints((P, N), -16, 16, gen, torch.float32, "cuda")
    buf, out = guarded(groups * (P + 1), N, torch.bfloat16, "cuda")
    L.gemm_tile(a, w, out, bias, rows_per_group=P, group_stride=P + 1, group_offset=1, row_add=row_add, tile_n=tile_n)
    torch.cuda.synchronize()
    assert_guard(buf, out, "row remap")
    ref, _ = gemm_ref(a, w, bias)
    ref = ref.view(groups, P, N) + row_add.double()
    got = out.view(groups, P + 1, N)
    assert_exact(got[:, 1:].reshape(M, N), ref.reshape(M, N), "row remap tile %d" % tile_n)
    it, pat = H.SENTINEL[torch.bfloat16]
    assert bool((got[:, 0].contiguous().view(it) == pat).all()), "a class-token row was overwritten"


BENCH_SHAPES = [  # (M, N, K, act, residual, dispatched width on 132 SMs) of the default benchmark workload
    (19456, 37888, 3584, ACT_SWIGLU, False, 256), (19456, 3584, 18944, ACT_NONE, True, 256),
    (50176, 3840, 1280, ACT_NONE, False, 128),
]


@pytest.mark.parametrize("M,N,K,act,with_res,width", BENCH_SHAPES)
def test_dispatched_and_256_are_bit_identical_to_128(L, M, N, K, act, with_res, width):
    """Every output element is one accumulator summed over the k-blocks in order whatever the tile width, so neither the
    width the dispatcher picks nor a forced 256 changes a bit of the result."""
    if H._sms() == 132:
        assert tile_width(M, N, K, 132) == width
    gen = torch.Generator(device="cuda").manual_seed(K)
    a = torch.randn(M, K, device="cuda", generator=gen).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=gen) / K ** 0.5).bfloat16()
    n_out = N // 2 if act == ACT_SWIGLU else N
    res = torch.randn(M, n_out, device="cuda", generator=gen).bfloat16() if with_res else None
    outs = [L.gemm_tile(a, w, torch.empty(M, n_out, device="cuda", dtype=torch.bfloat16), residual=res, act=act, tile_n=t)
            for t in (128, 0, 256)]
    torch.cuda.synchronize()
    assert torch.equal(outs[1], outs[0]) and torch.equal(outs[2], outs[0])
