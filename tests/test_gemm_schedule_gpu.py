"""GPU tests of the GEMM's persistent schedule: the two MMA warpgroups take alternate tiles of each CTA and the tiles
are walked in groups of 32 M-tiles.  The shapes put the schedule's boundaries under test: CTAs with an odd number of
tiles or with one tile (one warpgroup idle), mainloops shorter than an epilogue, ragged edges, a ragged last M group,
and every compiled epilogue class with several tiles per CTA.

Reference = torch fp32 on the bf16-rounded inputs, at the tolerances of test_kernels_gpu.py.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF_RTOL, BF_ATOL = 1.0e-2, 2e-2      # bf16 outputs
F32_RTOL, F32_ATOL = 1e-4, 1e-3      # fp32 outputs


def dev():
    return torch.device("cuda:0")


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev()).to(torch.bfloat16)


def assert_close(got, ref, rtol, atol, what=""):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    bad = (err > atol + rtol * ref.abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} outside tol, max err {err.max().item():.4e}"


def gelu_grad(z):
    return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


# (M, N) with M, N multiples of 128: tile count = M/128 * N/128.  132 is the H100's SM count, so 131-133 and 263-265
# give CTAs with one tile, two tiles and an odd number of tiles.
@pytest.mark.parametrize("tm,tn", [(1, 1), (1, 131), (12, 11), (7, 19), (1, 263), (12, 22), (5, 53)])
def test_tile_counts(tm, tn):
    from otter_b200 import functional as F
    x, w = rnd(128 * tm, 256), rnd(128 * tn, 256, scale=0.1)
    assert_close(F.linear_fwd(x, w), x.float() @ w.float().t(), BF_RTOL, BF_ATOL, f"{tm * tn} tiles")


# K = 16 / 64 / 72: one (partial) k-block, far shorter than the other warpgroup's epilogue; K = 16384: 256 k-blocks
@pytest.mark.parametrize("K", [16, 64, 72, 16384])
def test_depths(K):
    from otter_b200 import functional as F
    x, w = rnd(2048, K), rnd(4096, K, scale=K ** -0.5)
    z = torch.empty(2048, 4096, device=dev(), dtype=torch.bfloat16)
    h = F.linear_fwd(x, w, act=1, aux_out=z)
    zr = x.float() @ w.float().t()
    assert_close(z, zr, BF_RTOL, BF_ATOL, f"aux_out K={K}")
    assert_close(h, torch.nn.functional.gelu(zr), BF_RTOL, BF_ATOL, f"gelu K={K}")


def test_ragged_edges():
    from otter_b200 import functional as F
    M, N, K = 2056, 1032, 1024                 # M = 16 * 128 + 8, N = 8 * 128 + 8
    x, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    assert_close(F.linear_fwd(x, w), x.float() @ w.float().t(), BF_RTOL, BF_ATOL, "fwd")
    dy = rnd(M, N)
    w2 = rnd(N, K, scale=N ** -0.5)
    assert_close(F.linear_dgrad(dy, w2), dy.float() @ w2.float(), BF_RTOL, BF_ATOL, "dgrad")
    assert_close(F.linear_wgrad(dy, x), dy.float().t() @ x.float(), F32_RTOL, F32_ATOL, "wgrad")


# M = 16520: 130 M-tiles = 4 full groups of 32 and a last group of 2, the last M-tile itself partial
@pytest.mark.parametrize("layout", ["fwd", "dgrad", "wgrad"])
def test_grouped_walk_ragged_last_group(layout):
    from otter_b200 import functional as F
    M, N, K = 16520, 384, 256
    if layout == "fwd":
        x, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
        assert_close(F.linear_fwd(x, w), x.float() @ w.float().t(), BF_RTOL, BF_ATOL, layout)
    elif layout == "dgrad":
        dy, w = rnd(M, K), rnd(K, N, scale=K ** -0.5)
        assert_close(F.linear_dgrad(dy, w), dy.float() @ w.float(), BF_RTOL, BF_ATOL, layout)
    else:
        dy, x = rnd(K, M), rnd(K, N)
        assert_close(F.linear_wgrad(dy, x), dy.float().t() @ x.float(), F32_RTOL, F32_ATOL, layout)


# every compiled epilogue class (kEpiCls in otb_gemm.cu), and the run-time epilogue options with each combination the
# hot path uses outside those classes: fp32 residual (fp32-grade forward), bias + relu^2 + pre-activation (Persimmon
# up-projection), relu^2'(aux) (Persimmon dgrad), bias + GELU into fp32 (fp32-grade forward); at 8 x 64 = 512 tiles
@pytest.mark.parametrize("cls", list(range(14)) + ["res_fp32", "relu2_aux_out", "relu2_grad", "gelu_f32"])
def test_epilogue_classes(cls):
    from otter_b200 import functional as F
    M, N, K = 1024, 8192, 128
    x, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    zr = x.float() @ w.float().t()
    gate = torch.tensor([0.5], device=dev())
    g = math.tanh(0.5)
    bias = torch.randn(N, device=dev(), generator=torch.Generator(device=dev()).manual_seed(5))
    res = rnd(M, N, seed=7)
    aux = (zr + 0.1).to(torch.bfloat16)
    bf, f32 = (BF_RTOL, BF_ATOL), (F32_RTOL, F32_ATOL)
    z = torch.empty(M, N, device=dev(), dtype=torch.bfloat16)
    if cls == 0:
        got, ref, tol = F.linear_fwd(x, w), zr, bf
    elif cls == 1:
        got, ref, tol = F.linear_fwd(x, w, scale_ptr=gate, scale_tanh=True), zr * g, bf
    elif cls == 2:
        got, ref, tol = F.linear_fwd(x, w, bias=bias), zr + bias, bf
    elif cls == 3:
        zz = zr + bias
        got, ref, tol = F.linear_fwd(x, w, bias=bias, act=2), zz * torch.sigmoid(1.702 * zz), bf
    elif cls == 4:
        got, ref, tol = F.linear_fwd(x, w, bias=bias, residual=res), zr + bias + res.float(), bf
    elif cls == 5:
        got, ref, tol = F.linear_fwd(x, w, residual=res), zr + res.float(), bf
    elif cls == 6:
        got, ref, tol = F.linear_fwd(x, w, act=1, aux_out=z), torch.nn.functional.gelu(zr), bf
        assert_close(z, zr, *bf, "aux_out")
    elif cls == 7:
        got = F.linear_fwd(x, w, aux_out=z, scale_ptr=gate, scale_tanh=True, residual=res)
        ref, tol = zr * g + res.float(), bf
        assert_close(z, zr, *bf, "aux_out")
    elif cls == 8:
        got = F.linear_fwd(x, w, aux_in=aux, scale_ptr=gate, scale_tanh=True)
        ref, tol = zr * gelu_grad(aux.float()) * g, bf
    elif cls == 9:
        got, ref, tol = F.linear_fwd(x, w, aux_in=aux), zr * gelu_grad(aux.float()), bf
    elif cls == 10:
        got, ref, tol = F.linear_fwd(x, w, out_dtype=torch.float32), zr, f32
    elif cls == 11:
        got = F.linear_fwd(x, w, out_dtype=torch.float32, scale_ptr=gate, scale_tanh=True)
        ref, tol = zr * g, f32
    elif cls in (12, 13):
        old = torch.randn(M, N, device=dev(), generator=torch.Generator(device=dev()).manual_seed(9))
        epi = dict(scale_ptr=gate, scale_tanh=True) if cls == 13 else {}
        got = F._gemm_raw(x, 0, x.stride(0), w, 0, w.stride(0), M, N, K, old.clone(), accumulate=True, **epi)
        ref, tol = old + zr * (g if cls == 13 else 1.0), f32
    elif cls == "res_fp32":
        res32 = torch.randn(M, N, device=dev(), generator=torch.Generator(device=dev()).manual_seed(11))
        out = torch.empty(M, N, device=dev())
        got = F._gemm_raw(x, 0, x.stride(0), w, 0, w.stride(0), M, N, K, out, residual=res32, res_fp32=True)
        ref, tol = zr + res32, f32
    elif cls == "relu2_aux_out":
        got, ref, tol = F.linear_fwd(x, w, bias=bias, act=3, aux_out=z), torch.relu(zr + bias) ** 2, bf
        assert_close(z, zr + bias, *bf, "aux_out")
    elif cls == "relu2_grad":
        got, ref, tol = F.linear_fwd(x, w, aux_in=aux, act=3), zr * 2 * torch.relu(aux.float()), bf
    else:
        got = F.linear_fwd(x, w, bias=bias, act=1, out_dtype=torch.float32)
        ref, tol = torch.nn.functional.gelu(zr + bias), f32
    assert_close(got, ref, *tol, f"class {cls}")


def test_bit_identical_runs_and_accumulate_twice():
    from otter_b200 import functional as F
    x, w = rnd(2048, 4096), rnd(16384, 4096, scale=4096 ** -0.5)
    z1 = torch.empty(2048, 16384, device=dev(), dtype=torch.bfloat16)
    z2 = torch.empty_like(z1)
    h1 = F.linear_fwd(x, w, act=1, aux_out=z1)
    h2 = F.linear_fwd(x, w, act=1, aux_out=z2)
    assert torch.equal(h1, h2) and torch.equal(z1, z2)
    dz, xa = rnd(2048, 16384), rnd(2048, 4096)
    gw = torch.zeros(16384, 4096, device=dev())
    F.linear_wgrad(dz, xa, out=gw, accumulate=True)
    once = gw.clone()
    F.linear_wgrad(dz, xa, out=gw, accumulate=True)
    assert_close(once, dz.float().t() @ xa.float(), F32_RTOL, 2e-3, "wgrad_up accumulate once")
    assert_close(gw, 2 * once, F32_RTOL, 2e-3, "accumulate twice")
