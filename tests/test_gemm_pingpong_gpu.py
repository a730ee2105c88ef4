"""Normal-mode GEMM (n_tok > 64: two consumer warpgroups alternating the tiles of each persistent CTA, epilogue from the
accumulator registers) against the fp32 restatement, at the shapes its schedule can get wrong: tile counts around the SM
count, odd / even tiles per CTA, M / N / K tails, every epilogue, in-place residual, repeated launches."""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
BF16_RTOL = 2 ** -7  # one bf16 ulp, as in test_kernels_gpu.py
# GELU after the bf16 rounding of the linear output: where that rounding goes the other way (fp32 summation order), the
# second rounding can make it two ulps -- rare, but millions of elements meet it
GELU_RTOL = 2 * BF16_RTOL
SUM_RTOL = 2 * BF16_RTOL  # residual add after that rounding (see _close_sum)


@pytest.fixture(scope="module")
def ops():
    from audio_flamingo_b200 import ops as _ops

    return _ops


def _rand(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(bf16).cuda()


def _close(got, ref, rtol, atol, what=""):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    bad = (err > atol + rtol * ref.abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} out of tolerance, max err {err.max().item():.4g}"


def _close_sum(got, ref, parts, rtol, atol, what=""):
    """ref = bf16(sum of parts): an ulp of a part rounded the other way survives where the parts cancel, and the sum is
    rounded once more, so the tolerance scales with the parts' magnitudes, not the result's (as
    test_gemm_splitk_deterministic_and_epilogue does): |err| <= ulp(part) + ulp(sum) <= 2 * 2^-7 * sum |part|."""
    err = (got.float() - ref.float()).abs()
    tol = atol + rtol * sum(p.float().abs() for p in parts)
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} out of tolerance, max err {err.max().item():.4g}"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("extra", [-1, 0, 1])
def test_tile_count_around_sm_count(ops, extra):
    """One 128-column tile per row tile: sm_count - 1, sm_count and sm_count + 1 tiles."""
    M, N, K = 128 * (_sms() + extra), 128, 64
    x, w, b = _rand((M, K), 1.0, 1), _rand((N, K), 0.1, 2), _rand((N,), 0.5, 3)
    _close(ops.linear(x, w, b), (x.float() @ w.float().T + b.float()).to(bf16), BF16_RTOL, 1e-3, f"tiles {M // 128}")


@pytest.mark.parametrize("per_cta", [2, 3, 4, 5])
def test_odd_and_even_tiles_per_cta(ops, per_cta):
    """With an odd number of tiles per CTA the first consumer warpgroup runs one tile more than the second."""
    M, N, K = 128 * _sms(), 128 * per_cta, 192
    x, w, b = _rand((M, K), 1.0, 4), _rand((N, K), 0.08, 5), _rand((N,), 0.5, 6)
    _close(ops.linear(x, w, b, gelu=True), torch.nn.functional.gelu((x.float() @ w.float().T + b.float()).to(bf16).float()).to(bf16),
           GELU_RTOL, 2e-3, f"{per_cta} tiles per CTA")


@pytest.mark.parametrize("M", [130, 257])
@pytest.mark.parametrize("N", [100, 200, 384])
@pytest.mark.parametrize("K", [64, 136, 1000])
def test_tails(ops, M, N, K):
    """M and N tails (N = 100: output rows not 16-byte aligned -> direct stores), K not a multiple of 64."""
    x, w, b = _rand((M, K), 1.0, 7), _rand((N, K), 0.05, 8), _rand((N,), 0.5, 9)
    ref = (x.float() @ w.float().T + b.float()).to(bf16)
    _close(ops.linear(x, w, b), ref, BF16_RTOL, 1e-3, f"bias {M}x{N}x{K}")
    res = _rand((M, N), 1.0, 10)
    _close_sum(ops.linear(x, w, b, resid=res), (ref.float() + res.float()).to(bf16), (ref, res), SUM_RTOL, 4e-3, f"bias+resid {M}x{N}x{K}")


@pytest.mark.parametrize("M,N,K", [(640, 512, 256), (1000, 1280, 1280)])
def test_every_epilogue(ops, M, N, K):
    x, w, b = _rand((M, K), 1.0, 11), _rand((N, K), K ** -0.5, 12), _rand((N,), 0.5, 13)
    res = _rand((M, N), 1.0, 14)
    acc = x.float() @ w.float().T
    lin = (acc + b.float()).to(bf16)
    gelu = torch.nn.functional.gelu(lin.float()).to(bf16)
    _close(ops.linear(x, w), acc.to(bf16), BF16_RTOL, 1e-3, "plain")
    _close(ops.linear(x, w, b), lin, BF16_RTOL, 1e-3, "bias")
    _close(ops.linear(x, w, b, gelu=True), gelu, GELU_RTOL, 2e-3, "bias+gelu")
    plain = acc.to(bf16)
    _close_sum(ops.linear(x, w, b, resid=res), (lin.float() + res.float()).to(bf16), (lin, res), SUM_RTOL, 4e-3, "bias+resid")
    _close_sum(ops.linear(x, w, resid=res), (plain.float() + res.float()).to(bf16), (plain, res), SUM_RTOL, 4e-3, "resid")
    # in place (o_proj / down / out_proj / fc2): out is the residual
    h = res.clone()
    ops.linear(x, w, b, resid=h, out=h)
    _close_sum(h, (lin.float() + res.float()).to(bf16), (lin, res), SUM_RTOL, 4e-3, "bias+resid in place")
    h = res.clone()
    ops.linear(x, w, resid=h, out=h)
    _close_sum(h, (plain.float() + res.float()).to(bf16), (plain, res), SUM_RTOL, 4e-3, "resid in place")
    # bias + GELU + periodic residual (conv2 + positional embedding)
    period = 24
    pos = _rand((period, N), 1.0, 15)
    rows = torch.arange(M, device="cuda") % period
    _close_sum(ops.linear(x, w, b, gelu=True, resid=pos, res_period=period), (gelu.float() + pos.float()[rows]).to(bf16),
               (gelu, pos[rows]), GELU_RTOL + BF16_RTOL, 4e-3, "bias+gelu+pos")
    # fp32 output (direct stores)
    out = ops.linear(x, w, b, out_f32=True)
    assert out.dtype == torch.float32
    _close(out, lin.float(), BF16_RTOL, 1e-3, "f32out")
    # a flag set without a compile-time specialisation (generic instantiation): GELU without bias
    _close(ops.linear(x, w, gelu=True), torch.nn.functional.gelu(acc.to(bf16).float()).to(bf16), GELU_RTOL, 2e-3, "gelu, no bias")


@pytest.mark.parametrize("M,F", [(300, 384), (1000, 18944 // 37)])
def test_swiglu_both_layouts_long_k(ops, M, F):
    """SwiGLU at the decoder's K = 3584, interleaved (pack_gate_up) and [gate; up] layouts: same arithmetic, same bits."""
    K = 3584
    x, g, u = _rand((M, K), 1.0, 16), _rand((F, K), K ** -0.5, 17), _rand((F, K), K ** -0.5, 18)
    out = ops.swiglu_linear(x, ops.pack_gate_up(g, u), F)
    gate = (x.float() @ g.float().T).to(bf16)
    up = (x.float() @ u.float().T).to(bf16)
    ref = (torch.nn.functional.silu(gate.float()).to(bf16).float() * up.float()).to(bf16)
    _close(out, ref, 2 * BF16_RTOL, 2e-3, f"swiglu M={M} F={F}")
    if F % 128 == 0:
        assert torch.equal(ops.swiglu_linear(x, torch.cat([g, u], 0).contiguous(), F, concat=True), out)


def test_repeated_launches_bit_identical(ops):
    M, N, K = 128 * _sms() * 2 + 77, 1280, 1280  # several tiles per CTA, a row tail
    x, w, b = _rand((M, K), 1.0, 19), _rand((N, K), K ** -0.5, 20), _rand((N,), 0.5, 21)
    res = _rand((M, N), 1.0, 22)
    outs = [ops.linear(x, w, b, gelu=True) for _ in range(3)]
    outs_r = [ops.linear(x, w, b, resid=res) for _ in range(3)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    for o in outs_r[1:]:
        assert torch.equal(o, outs_r[0])
