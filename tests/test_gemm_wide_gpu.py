"""Wide normal-mode GEMM (K >= 2048: 128 x 256 tiles, the two consumer warpgroups share each tile, one m64n256k16 per k16
step) against the fp32 restatement, at the shapes its schedule can get wrong: odd and even row-tile counts, tile counts
around the SM count, M / N / K tails, every epilogue it takes, both SwiGLU layouts, repeated launches and programmatic
dependent launch.  Tolerances as in test_gemm_pingpong_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
BF16_RTOL = 2 ** -7
GELU_RTOL = 2 * BF16_RTOL
SUM_RTOL = 2 * BF16_RTOL
K_WIDE = 3584  # the decoder's hidden size: every epilogue takes the wide kernel at this K


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
    err = (got.float() - ref.float()).abs()
    tol = atol + rtol * sum(p.float().abs() for p in parts)
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} out of tolerance, max err {err.max().item():.4g}"


def _kernels(fn):
    """Names of the CUDA kernels fn launches."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_dispatch(ops):
    """K >= 2048 takes the wide kernel; small K and the periodic residual (conv2) keep the 128 x 128 ping-pong kernel."""
    x, w = _rand((1000, K_WIDE), 1.0, 1), _rand((1024, K_WIDE), K_WIDE ** -0.5, 2)
    wide = lambda names: any("gemm_tok_wide_kernel" in n for n in names)  # noqa: E731
    assert wide(_kernels(lambda: ops.linear(x, w)))
    assert wide(_kernels(lambda: ops.swiglu_linear(x, w, 512, concat=True)))
    pos = _rand((24, 1024), 1.0, 3)
    assert not wide(_kernels(lambda: ops.linear(x, w, resid=pos, res_period=24)))
    assert not wide(_kernels(lambda: ops.linear(x[:, :1280].contiguous(), w[:, :1280].contiguous())))


@pytest.mark.parametrize("row_tiles", [1, 2, 3, 7, 8])
def test_odd_and_even_row_tiles(ops, row_tiles):
    """Row tails: the last tile's rows past M read zeros and are not stored."""
    M, N = 128 * row_tiles - 5, 768
    x, w, b = _rand((M, K_WIDE), 1.0, 3), _rand((N, K_WIDE), K_WIDE ** -0.5, 4), _rand((N,), 0.5, 5)
    out = torch.full((M + 64, N), 7.0, device="cuda", dtype=bf16)  # rows past M must stay untouched
    ops.linear(x, w, b, out=out[:M])
    _close(out[:M], (x.float() @ w.float().T + b.float()).to(bf16), BF16_RTOL, 1e-3, f"{row_tiles} row tiles")
    assert torch.all(out[M:] == 7.0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("extra", [-1, 0, 1, None])
def test_tile_count_around_sm_count(ops, extra):
    """One 256-column tile per row tile: sm_count - 1, sm_count and sm_count + 1 tiles, and 2 sm_count + 1."""
    tiles = 2 * _sms() + 1 if extra is None else _sms() + extra
    M, N, K = 128 * tiles, 256, K_WIDE
    x, w = _rand((M, K), 1.0, 6), _rand((N, K), K ** -0.5, 7)
    _close(ops.linear(x, w), (x.float() @ w.float().T).to(bf16), BF16_RTOL, 1e-3, f"{tiles} tiles")


@pytest.mark.parametrize("M", [130, 300])
@pytest.mark.parametrize("N", [200, 384, 520])
@pytest.mark.parametrize("K", [K_WIDE, K_WIDE + 8])
def test_tails(ops, M, N, K):
    """M tails inside a tile, N not a multiple of 256, K not a multiple of 64."""
    x, w, b = _rand((M, K), 1.0, 8), _rand((N, K), K ** -0.5, 9), _rand((N,), 0.5, 10)
    ref = (x.float() @ w.float().T + b.float()).to(bf16)
    _close(ops.linear(x, w, b), ref, BF16_RTOL, 1e-3, f"bias {M}x{N}x{K}")
    res = _rand((M, N), 1.0, 11)
    _close_sum(ops.linear(x, w, b, resid=res), (ref.float() + res.float()).to(bf16), (ref, res), SUM_RTOL, 4e-3, f"bias+resid {M}x{N}x{K}")


@pytest.mark.parametrize("M,N", [(640, 768), (1000, 1344)])
def test_every_epilogue(ops, M, N):
    K = K_WIDE
    x, w, b = _rand((M, K), 1.0, 12), _rand((N, K), K ** -0.5, 13), _rand((N,), 0.5, 14)
    res = _rand((M, N), 1.0, 15)
    acc = x.float() @ w.float().T
    lin = (acc + b.float()).to(bf16)
    plain = acc.to(bf16)
    gelu = torch.nn.functional.gelu(lin.float()).to(bf16)
    _close(ops.linear(x, w), plain, BF16_RTOL, 1e-3, "plain")
    _close(ops.linear(x, w, b), lin, BF16_RTOL, 1e-3, "bias")
    _close(ops.linear(x, w, b, gelu=True), gelu, GELU_RTOL, 2e-3, "bias+gelu")
    _close_sum(ops.linear(x, w, b, resid=res), (lin.float() + res.float()).to(bf16), (lin, res), SUM_RTOL, 4e-3, "bias+resid")
    h = res.clone()
    ops.linear(x, w, b, resid=h, out=h)
    _close_sum(h, (lin.float() + res.float()).to(bf16), (lin, res), SUM_RTOL, 4e-3, "bias+resid in place")
    h = res.clone()
    ops.linear(x, w, resid=h, out=h)
    _close_sum(h, (plain.float() + res.float()).to(bf16), (plain, res), SUM_RTOL, 4e-3, "resid in place")
    _close_sum(ops.linear(x, w, b, gelu=True, resid=res), (gelu.float() + res.float()).to(bf16), (gelu, res),
               GELU_RTOL + BF16_RTOL, 4e-3, "bias+gelu+resid")


@pytest.mark.parametrize("M,F", [(300, 384), (1000, 18944 // 37), (777, 200)])
def test_swiglu_both_layouts(ops, M, F):
    """Interleaved (pack_gate_up; F % 128 != 0 too) and [gate; up] layouts: same arithmetic, same bits."""
    K = K_WIDE
    x, g, u = _rand((M, K), 1.0, 17), _rand((F, K), K ** -0.5, 18), _rand((F, K), K ** -0.5, 19)
    out = ops.swiglu_linear(x, ops.pack_gate_up(g, u), F)
    gate = (x.float() @ g.float().T).to(bf16)
    up = (x.float() @ u.float().T).to(bf16)
    ref = (torch.nn.functional.silu(gate.float()).to(bf16).float() * up.float()).to(bf16)
    _close(out, ref, 2 * BF16_RTOL, 2e-3, f"swiglu M={M} F={F}")
    if F % 128 == 0:
        assert torch.equal(ops.swiglu_linear(x, torch.cat([g, u], 0).contiguous(), F, concat=True), out)


def test_repeated_launches_bit_identical(ops):
    M, N, K = 128 * 132 * 2 + 77, 1280, K_WIDE
    x, w, b = _rand((M, K), 1.0, 20), _rand((N, K), K ** -0.5, 21), _rand((N,), 0.5, 22)
    res = _rand((M, N), 1.0, 23)
    outs = [ops.linear(x, w, b, gelu=True) for _ in range(3)]
    outs_r = [ops.linear(x, w, b, resid=res) for _ in range(3)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    for o in outs_r[1:]:
        assert torch.equal(o, outs_r[0])


def test_pdl_on_and_off_bit_identical(ops):
    """A chain of dependent wide GEMMs with programmatic dependent launch on and off: each waits for its producer."""
    from audio_flamingo_b200 import _lib

    M, K, F = 3000, K_WIDE, K_WIDE
    x = _rand((M, K), 1.0, 24)
    wg = _rand((2 * F, K), K ** -0.5, 25)
    wd = _rand((K, F), F ** -0.5, 26)

    def chain():
        h = x.clone()
        for _ in range(3):
            a = ops.swiglu_linear(h, wg, F, concat=True)
            ops.linear(a, wd, resid=h, out=h)
        return h

    lib = _lib.load()
    try:
        lib.af3_set_pdl(1)
        on = chain()
        torch.cuda.synchronize()
    finally:
        lib.af3_set_pdl(0)
    off = chain()
    assert torch.equal(on, off)
