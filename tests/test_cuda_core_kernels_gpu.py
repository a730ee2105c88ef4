"""Every launch path of the CUDA-core kernels (elementwise.cu, logmel.cu) against plain torch restatements of the same op
with the reference's rounding points, at the shapes where each host function switches kernels and the inputs where such
kernels go wrong: row-count and dim thresholds, tails, sweeps, alignment, ties, non-finite values, negative maxima.

test_dispatch asserts which kernel each case runs (torch.profiler kernel names, every case in one profiler session: repeated
sessions in one process can come back empty), so that a later change to a dispatch threshold cannot quietly move a case onto
another path.

Tolerance rule.  A tolerance of one bf16 ulp cannot see a missing intermediate rounding: dropping one bf16 rounding point
moves an output by at most an ulp.  So every kernel with a rounded bf16 output gets two assertions:
  1. the error is within one bf16 ulp of the restatement (relative 2^-7, plus the absolute floor the older tests use);
  2. at least a stated fraction of the elements is bit-identical to it.  The remaining elements differ where rsqrt, cos / sin
     or a different summation order land next to a rounding tie.  Each floor sits below the fraction measured on an H100
     (quoted next to it) with margin.
Integer and copy kernels (scatter, argmax, im2col, gate/up packing) are compared with torch.equal."""
import json
import math
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
BF16_RTOL = 2 ** -7


@pytest.fixture(scope="module")
def ops():
    from audio_flamingo_b200 import ops as _ops

    return _ops


def _rand(shape, scale=1.0, seed=0, dtype=bf16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _kernels(fn):
    """Names of the CUDA kernels fn launches, in launch order.  fn must be repeatable: it launches at least one kernel, so a
    session that recorded none lost its activity records, and fn runs again under a new session."""
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if evs:
            break
    return [e.name for e in sorted(evs, key=lambda e: e.time_range.start)]


def _tmpl(name, *args):
    """Regex of a kernel name with template arguments, which may be printed with spaces (`<true, 5>`)."""
    return name + r"<\s*" + r"\s*,\s*".join(args) + r"\s*>"


def _close(got, ref, atol, what, rtol=BF16_RTOL):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    bad = (err > atol + rtol * ref.abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} out of tolerance, max err {err.max().item():.4g}"


def _exact(got, ref, floor, what):
    frac = (got == ref).float().mean().item()
    assert frac >= floor, f"{what}: bit-identical fraction {frac:.6f} < {floor}"


# ---------------------------------------------------------------------------------------------------- RMSNorm
def _rmsnorm_ref(x, w, eps):
    """Qwen2RMSNorm: h = x.float(); h = h * rsqrt(mean(h^2) + eps); weight * h.to(bf16)."""
    h = x.float()
    h = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + eps)
    return w * h.to(bf16)


def _row_idx(rows, seed):
    """A permutation of the rows with repeats."""
    idx = torch.randperm(rows, generator=torch.Generator(device="cpu").manual_seed(seed))
    idx[::7] = idx[3]
    return idx.to(torch.int32).cuda()


def _rmsnorm_path(rows, dim):
    if rows <= 1024:
        return r"rmsnorm_rowblock_kernel"
    need = -(-(dim // 8) // 32)
    return _tmpl(r"rmsnorm_kernel", "5" if need <= 5 else "14" if need <= 14 else "16")


RMS_DIMS, RMS_ROWS = [256, 1280, 1288, 3584, 3592, 4096], [1024, 1025, 4000]


@pytest.mark.parametrize("dim", RMS_DIMS)
@pytest.mark.parametrize("rows", RMS_ROWS)
def test_rmsnorm_paths(ops, rows, dim):
    """Both sides of the row-block threshold (rows <= 1024) and both edges of NV = 5 / 14 / 16; an all-zero row (output 0)
    and a row of magnitude 1e4; row_idx (a permutation with repeats) bit-identical to indexing the full output."""
    x, w = _rand((rows, dim), 3.0, 100 + dim), _rand((dim,), 1.0, 101)
    x[0] = 0
    x[1] = (x[1].float() * (1e4 / 3)).to(bf16)
    out = ops.rmsnorm(x, w, 1e-6)
    ref = _rmsnorm_ref(x, w, 1e-6)
    assert torch.isfinite(out.float()).all() and (out[0] == 0).all()
    # two chained roundings (bf16(h), then weight * h): where the fp32 sum of squares, added in another order, moves h across a
    # rounding tie, one ulp of h can become two ulps of the output
    _close(out, ref, 1e-3, f"rmsnorm {rows}x{dim}", rtol=2 * BF16_RTOL)
    _exact(out, ref, 0.9999, f"rmsnorm {rows}x{dim}")  # H100: >= 0.99999 (the row-block kernel: 1.0)
    idx = _row_idx(rows, rows + dim)
    assert torch.equal(ops.rmsnorm(x, w, 1e-6, row_idx=idx), out[idx.long()])


# ---------------------------------------------------------------------------------------------------- LayerNorm
def _ln_path(pool, dim):
    need = -(-(dim // 8) // 32)
    nv = next(v for v in (2, 5, 8, 16) if need <= v)
    return _tmpl(r"layernorm_kernel", "true" if pool else "false", str(nv))


def _ln_ref(x, g, b):
    return torch.nn.functional.layer_norm(x.float(), (x.shape[-1],), g.float(), b.float(), 1e-5).to(bf16)


LN_DIMS = [128, 512, 520, 1280, 1288, 2048, 2056, 4096]
POOL_CASES = [(51, d) for d in LN_DIMS] + [(1501, 1280), (50, 1280)]


@pytest.mark.parametrize("dim", LN_DIMS)
def test_layernorm_paths(ops, dim):
    """NV = 2 / 5 / 8 / 16 at both edges, 333 rows (not a multiple of the 8 rows per CTA); one row of 100 + noise, where a
    one-pass variance (E[x^2] - mean^2 in fp32) would lose about ten bits to cancellation and move a large share of the row."""
    rows = 333
    x, g, b = _rand((rows, dim), 2.0, 110 + dim), _rand((dim,), 1.0, 111), _rand((dim,), 0.3, 112)
    x[5] = (100.0 + _rand((dim,), 1.0, 113).float()).to(bf16)
    out = ops.layernorm(x, g, b)
    ref = _ln_ref(x, g, b)
    _close(out, ref, 4e-3, f"layernorm dim={dim}")
    _exact(out, ref, 0.999, f"layernorm dim={dim}")  # H100: >= 0.99996
    _exact(out[5], ref[5], 0.995, f"layernorm dim={dim}, row 100 + noise")  # H100: >= 0.9995 (one element of 2056)


@pytest.mark.parametrize("T,dim", POOL_CASES)
def test_avgpool_layernorm_paths(ops, T, dim):
    """AvgPool1d(2, 2) + LayerNorm over 3 windows: every NV edge; odd T drops each window's last frame, as AvgPool1d does."""
    n_win = 3
    x, g, b = _rand((n_win * T, dim), 2.0, 120 + T + dim), _rand((dim,), 1.0, 121), _rand((dim,), 0.3, 122)
    x[T - 1] = 1e4  # window 0's last frame: dropped when T is odd
    out = ops.avgpool_layernorm(x, n_win, T, g, b)
    assert out.shape == (n_win * (T // 2), dim)
    pooled = torch.nn.functional.avg_pool1d(x.view(n_win, T, dim).permute(0, 2, 1).float(), 2, 2).to(bf16).permute(0, 2, 1)
    ref = _ln_ref(pooled.reshape(-1, dim), g, b)
    _close(out, ref, 4e-3, f"avgpool+layernorm T={T} dim={dim}")
    _exact(out, ref, 0.999, f"avgpool+layernorm T={T} dim={dim}")  # H100: >= 0.99989


# ---------------------------------------------------------------------------------------------------- RoPE + KV append
def rope_reference(qkv, B, T, H, Hkv, D, pos0, inv_freq, kv_start=None):
    """Rotate-half RoPE ([O] Q2M:100-146) of the q and k heads of a packed [B*T, (H + 2 Hkv) * D] bf16 projection, every
    bf16 op of the reference rounded (fp32 cos / sin tables cast to bf16).  Slot pos0 + t of sequence b is at position
    slot - kv_start[b]; padded slots (negative position) take position 1 (GEN:721).  Returns (q, k, v) as [B, T, heads, D]."""
    slots = pos0 + torch.arange(T, device=qkv.device)[None, :]
    pos = slots - (kv_start.long()[:, None] if kv_start is not None else 0)
    pos = torch.where(pos < 0, torch.ones_like(pos), pos).expand(B, T).float()
    freqs = pos[:, :, None] * inv_freq[None, None, :]
    emb = torch.cat([freqs, freqs], -1)
    cos, sin = emb.cos().to(bf16)[:, :, None, :], emb.sin().to(bf16)[:, :, None, :]

    def rot(x):
        x1, x2 = x[..., : D // 2], x[..., D // 2:]
        return x * cos + torch.cat([-x2, x1], -1) * sin

    o = qkv.view(B, T, H + 2 * Hkv, D)
    return rot(o[:, :, :H]), rot(o[:, :, H:H + Hkv]), o[:, :, H + Hkv:]


def _inv_freq(D, theta=1e6):
    return (1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).cuda()


def _rope_run(ops, qkv, B, T, H, Hkv, D, Tmax, pos0, kv_start=None):
    """(rotated copy of qkv, k cache, v cache); the caches start filled with 3."""
    out = qkv.clone()
    k_cache = torch.full((B, Hkv, Tmax, D), 3.0, device="cuda", dtype=bf16)
    v_cache = torch.full_like(k_cache, 3.0)
    ops.rope_kv_append(out, k_cache, v_cache, B=B, T=T, H=H, Hkv=Hkv, D=D, pos0=pos0, inv_freq=_inv_freq(D), kv_start=kv_start)
    return out, k_cache, v_cache


ROPE_CASES = [
    (1, 1023, 1024, 0, None, True),                 # B*T*D/16 = 8184: head-parallel
    (1, 1024, 1024, 0, None, False),                # 8192: prefill kernel
    (2, 512, 1024, 512, [0, 700], False),           # continuation, left padding, last slot = Tmax - 1
    (3, 100, 1024, 924, [0, 950, 1023], True),      # the same in the head-parallel kernel
]


@pytest.mark.parametrize("B,T,Tmax,pos0,starts,head_par", ROPE_CASES)
def test_rope_kv_append_paths(ops, B, T, Tmax, pos0, starts, head_par):
    H, Hkv, D = 28, 4, 128
    orig = _rand((B * T, (H + 2 * Hkv) * D), 1.0, 130 + T)
    kv_start = torch.tensor(starts, dtype=torch.int32, device="cuda") if starts is not None else None
    got, kc, vc = _rope_run(ops, orig, B, T, H, Hkv, D, Tmax, pos0, kv_start)
    q_ref, k_ref, v_ref = rope_reference(orig, B, T, H, Hkv, D, pos0, _inv_freq(D), kv_start)
    got = got.view(B, T, H + 2 * Hkv, D)
    k_got, v_got = kc[:, :, pos0:pos0 + T].transpose(1, 2), vc[:, :, pos0:pos0 + T].transpose(1, 2)
    # a one-ulp difference of a bf16 cos / sin can survive the cancellation in x1 cos - x2 sin: absolute floor as in test_rope_kv_append
    _close(got[:, :, :H], q_ref, 2 ** -6 * q_ref.float().abs().max().item(), "rope q")
    _close(k_got, k_ref, 2 ** -6 * k_ref.float().abs().max().item(), "rope k")
    _exact(got[:, :, :H], q_ref, 0.9999, "rope q")  # H100: 1.0
    _exact(k_got, k_ref, 0.9999, "rope k")
    assert torch.equal(v_got, v_ref)
    assert torch.equal(got[:, :, H:], orig.view(B, T, H + 2 * Hkv, D)[:, :, H:]), "k / v heads of the projection must stay"
    outside = torch.ones(Tmax, dtype=torch.bool)
    outside[pos0:pos0 + T] = False
    assert (kc[:, :, outside] == 3).all() and (vc[:, :, outside] == 3).all(), "slots outside [pos0, pos0 + T) must stay"


def test_rope_kv_append_paths_agree(ops):
    """The head-parallel kernel on 1023 tokens and the prefill kernel on the same tokens plus one: identical bits on the rows
    they share (queries and both caches)."""
    H, Hkv, D, Tmax = 28, 4, 128, 1024
    qkv = _rand((1024, (H + 2 * Hkv) * D), 1.0, 140)
    part, kp, vp = _rope_run(ops, qkv[:1023], 1, 1023, H, Hkv, D, Tmax, 0)
    full, kf, vf = _rope_run(ops, qkv, 1, 1024, H, Hkv, D, Tmax, 0)
    assert torch.equal(part, full[:1023])
    assert torch.equal(kp[:, :, :1023], kf[:, :, :1023]) and torch.equal(vp[:, :, :1023], vf[:, :, :1023])


# ---------------------------------------------------------------------------------------------------- embed scatter
_POST = [48, 60, 0, 13, 48, 100, 0, 7, 48, 31, 48, 48, 0, 22, 48, 5, 48, 70, 19, 48]  # 20 windows: clamped (> 48) and empty ones
_FRAMES = 48
_N_VALID = sum(min(p, _FRAMES) for p in _POST)  # 625


def _scatter_case(ops, n_tok, runs, seed):
    V, dim, n_win = 1000, 64, len(_POST)
    aid = V - 1
    table, audio = _rand((V, dim), 1.0, seed), _rand((n_win * _FRAMES, dim), 1.0, seed + 1)
    post = torch.tensor(_POST, dtype=torch.int32, device="cuda")
    g = torch.Generator().manual_seed(seed + 2)
    ids = torch.randint(0, V - 1, (n_tok,), generator=g)
    for a, b in runs:
        ids[a:b] = aid
    ids = ids.cuda()
    out, counts = ops.embed_scatter(ids, table, aid, audio, n_win, _FRAMES, post)
    valid = (torch.arange(_FRAMES, device="cuda")[None, :] < post[:, None]).reshape(-1)
    return ids == aid, table[ids], audio[valid], out, counts


SCATTER_CASES = [
    (1024, [(200, 500), (699, 1024)]),            # one sweep of 1024 ids
    (1025, [(100, 300), (600, 1025)]),            # two sweeps; the second run crosses 1024
    (3000, [(900, 1100), (1900, 2325)]),          # three sweeps; runs cross 1024 and 2048
]


@pytest.mark.parametrize("n_tok,runs", SCATTER_CASES)
def test_embed_scatter_sweeps(ops, n_tok, runs):
    """Audio-token ordinals carried across the 1024-id sweeps, the window search over 20 windows (empty and clamped ones
    included): bit-exact."""
    is_audio, ref, rows, out, counts = _scatter_case(ops, n_tok, runs, 150 + n_tok)
    assert sum(b - a for a, b in runs) == _N_VALID
    ref[is_audio] = rows
    assert torch.equal(out, ref)
    assert counts.tolist() == [_N_VALID, _N_VALID]


def test_embed_scatter_more_tokens_than_rows(ops):
    """More audio tokens than valid rows: counts disagree (the caller raises, as masked_scatter would); the first rows are
    still placed exactly and text rows are untouched."""
    runs = [(900, 1100), (1900, 2400)]
    is_audio, ref, rows, out, counts = _scatter_case(ops, 3000, runs, 160)
    n_audio = sum(b - a for a, b in runs)
    assert counts.tolist() == [n_audio, _N_VALID] and n_audio > _N_VALID
    pos = is_audio.nonzero().squeeze(1)
    assert torch.equal(out[pos[:_N_VALID]], rows)
    assert torch.equal(out[~is_audio], ref[~is_audio])


# ---------------------------------------------------------------------------------------------------- argmax
def _argmax_rows(B, V, seed):
    """Random logits with, row by row, the maximum first, last, tied across a slice boundary, an all -inf row, +inf entries,
    an all-equal row, and plain random rows."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn((B, V), generator=g)
    per = ((V + 31) // 32 + 3) & ~3  # the kernel's slice length
    for r in range(B):
        kind = (r + V) % 8
        if kind == 0:
            x[r, 0] = 60.0
        elif kind == 1:
            x[r, V - 1] = 60.0
        elif kind == 2 and V > per:
            s = min(3, (V - 1) // per - 1)
            x[r, (s + 1) * per - 1] = x[r, (s + 1) * per] = 60.0
        elif kind == 3:
            x[r] = -math.inf
        elif kind == 4:
            x[r, V // 2] = math.inf
            x[r, V - 1] = math.inf
        elif kind == 5:
            x[r] = 0.5
    return x.cuda()


ARGMAX_B, ARGMAX_V = [1, 33, 64], [1, 5, 127, 128, 2048, 152064, 152065]


@pytest.mark.parametrize("B", ARGMAX_B)
@pytest.mark.parametrize("V", ARGMAX_V)
def test_argmax_paths(ops, V, B):
    """V below the 32 slices (empty slices), V % 4 != 0 (rows not 16-byte aligned: scalar loads), ties across slices, non-finite
    rows: exactly torch.argmax (first maximal index)."""
    logits = _argmax_rows(B, V, 170 + V + B)
    got = ops.argmax(logits)
    if V % 4 and B > 1:
        assert (logits.data_ptr() + V * 4) % 16, "row 1 must take the scalar path"
    assert torch.equal(got, logits.argmax(-1))


def test_argmax_ignores_nan(ops):
    """NaN entries are skipped (unlike torch.argmax, which returns a NaN's index); an all-NaN row yields 0."""
    V = 152064
    logits = _argmax_rows(4, V, 180)
    logits[0, 0] = math.nan
    logits[1, 7] = 80.0
    logits[1, 100] = math.nan
    logits[2, 5000:6000] = math.nan
    logits[3] = math.nan
    got = ops.argmax(logits)
    want = torch.where(logits.isnan(), -math.inf, logits).argmax(-1)
    assert want[3].item() == 0 and want[1].item() == 7
    assert torch.equal(got, want)
    assert not torch.equal(got, logits.argmax(-1))


# ---------------------------------------------------------------------------------------------------- conv stem, gate/up packing
CONV1_T, CONV2_T = [1, 63, 64, 65, 3000], [1, 2, 63, 65, 1501]


@pytest.mark.parametrize("dtype", [torch.float32, bf16])
@pytest.mark.parametrize("T", CONV1_T)
def test_im2col_conv1_paths(ops, T, dtype):
    n_win, C = 2, 128
    x = _rand((n_win, C, T), 1.0, 190 + T, torch.float32).to(dtype)
    cols = ops.im2col_conv1(x)
    xp = torch.nn.functional.pad(x.to(bf16), (1, 1))
    ref = torch.stack([xp[:, :, kk:kk + T] for kk in range(3)], dim=1).permute(0, 3, 1, 2).reshape(n_win * T, 3 * C)
    assert torch.equal(cols, ref)


@pytest.mark.parametrize("T", CONV2_T)
def test_im2col_conv2_odd_t(ops, T):
    n_win, C = 3, 64
    h = _rand((n_win * T, C), 1.0, 200 + T)
    cols = ops.im2col_conv2(h, n_win, T)
    T_out = (T - 1) // 2 + 1
    hp = torch.nn.functional.pad(h.view(n_win, T, C), (0, 0, 1, 1))
    ref = torch.stack([hp[:, kk:kk + 2 * T_out:2, :] for kk in range(3)], dim=2).reshape(n_win * T_out, 3 * C)
    assert torch.equal(cols, ref)


@pytest.mark.parametrize("F", [200, 18944])
def test_pack_gate_up_layout(ops, F):
    """Per 128 features: 128 gate rows, then 128 up rows; rows past F are zero."""
    K = 256
    gate, up = _rand((F, K), 1.0, 210), _rand((F, K), 1.0, 211)
    packed = ops.pack_gate_up(gate, up)
    nb = -(-F // 128)
    gp, upp = torch.zeros((nb * 128, K), device="cuda", dtype=bf16), torch.zeros((nb * 128, K), device="cuda", dtype=bf16)
    gp[:F], upp[:F] = gate, up
    ref = torch.stack([gp.view(nb, 128, K), upp.view(nb, 128, K)], 1).reshape(2 * nb * 128, K)
    assert torch.equal(packed, ref)


# ---------------------------------------------------------------------------------------------------- log-mel
def logmel_reference(wave, filt):
    """fp64 restatement of WhisperFeatureExtractor's log-mel (WFE:135-164, exact DFT): wave float32 numpy [n_win, n_samples],
    filt [201, 128] -> [n_win, 128, n_samples // 160]."""
    win = torch.hann_window(400, dtype=torch.float64)
    st = torch.stft(torch.from_numpy(wave).double(), 400, 160, window=win, return_complex=True)
    mag = st[..., :-1].abs() ** 2
    mel = torch.from_numpy(filt).double().T @ mag
    ls = torch.clamp(mel, min=1e-10).log10()
    mx = ls.amax(dim=(1, 2), keepdim=True)
    return ((torch.maximum(ls, mx - 8.0) + 4.0) / 4.0).numpy()


def _mel_filters():
    from transformers.audio_utils import mel_filter_bank

    return mel_filter_bank(num_frequency_bins=201, num_mel_filters=128, min_frequency=0.0, max_frequency=8000.0,
                           sampling_rate=16000, norm="slaney", mel_scale="slaney")


def test_logmel_silent_quiet_and_tail(ops):
    """n_samples = 80 000 (500 frames: the last CTA holds 52 of its 64), five windows: silence (every output -1.5), quiet noise
    (the window maximum of log10 is negative, so the order-preserving int under atomicMax decides it), a quiet tone, loud noise,
    and a clip that turns silent half-way.  Same 1e-4 bound as the 30 s test."""
    filt = _mel_filters()
    tables = ops.LogMelTables(filt, "cuda")
    n = 80000
    rs = np.random.RandomState(7)
    wave = np.zeros((5, n), dtype=np.float32)
    wave[1] = rs.randn(n) * 1e-4
    wave[2] = 3e-4 * np.sin(2 * np.pi * 440.0 * np.arange(n) / 16000)
    wave[3] = rs.randn(n) * 0.3
    wave[4, : n // 2] = rs.randn(n // 2) * 0.05
    got = ops.logmel(torch.from_numpy(wave).cuda(), tables).cpu().numpy()
    ref = logmel_reference(wave, filt)
    assert got.shape == (5, 128, 500)
    assert np.abs(got[0] + 1.5).max() < 1e-6
    assert ref[1].max() * 4 - 4 < 0 and ref[2].max() * 4 - 4 < 0, "quiet windows must have a negative log10 maximum"
    err = np.abs(got - ref)
    assert err.max() < 1e-4, [float(e) for e in err.max(axis=(1, 2))]


# ---------------------------------------------------------------------------------------------------- Music Flamingo rotary time
def _rotary_time_ref(x, ts, inv_freq, W, T, window_duration, max_len):
    """MusicFlamingoRotaryEmbedding.forward + apply_rotary_time_emb ([O] musicflamingo/modular_musicflamingo.py:167-227):
    fp32 angles in the reference's operation order, fp32 cos / sin, the rotation of interleaved pairs in fp64, one rounding."""
    full = lambda t, v: torch.full_like(t, v)  # noqa: E731  (tensor divisors: torch turns a scalar divisor into a reciprocal multiply)
    wpos = torch.round(ts[:, 0] / full(ts[:, 0], window_duration))
    wpos = wpos / full(wpos, max_len)
    wf = torch.repeat_interleave(wpos[:, None] * inv_freq, 2, dim=-1)[:, None, :].expand(W, T, -1)
    positions = torch.arange(T, device=ts.device, dtype=torch.float32)
    positions = positions / full(positions, max_len) * (2 * math.pi)
    tf = torch.repeat_interleave(positions[:, None] * inv_freq, 2, dim=-1)[None].expand(W, T, -1)
    freqs = torch.cat((wf, tf), -1) * (-ts * 2 * math.pi)[..., None]
    cos, sin = freqs.cos().double(), freqs.sin().double()
    h = x.view(W, T, -1).double()
    rd = cos.shape[-1]
    r = h[..., :rd]
    pairs = r.reshape(W, T, -1, 2)
    rh = torch.stack((-pairs[..., 1], pairs[..., 0]), -1).flatten(-2)
    return torch.cat((r * cos + rh * sin, h[..., rd:]), -1).to(bf16).reshape(W * T, -1)


def test_rotary_time_embedding(ops):
    """Three windows at window indices 1, 2, 5 (non-zero window rotation), T = 300 (not a multiple of 256), dim 64 > 4 n_freq = 48:
    the 16 untouched features stay bit-identical."""
    W, T, dim, n_freq, step, max_len = 3, 300, 64, 12, 0.04, 1200
    window_duration = step * T
    k = torch.tensor([1.0, 2.0, 5.0])
    ts = (k[:, None] * T * step + torch.arange(T, dtype=torch.float32)[None, :] * step).float().cuda().contiguous()
    inv_freq = (1.0 / (10000 ** (torch.arange(0, 2 * n_freq, 2, dtype=torch.float32) / (2 * n_freq)))).cuda()
    orig = _rand((W * T, dim), 1.0, 220)
    x = ops.rotary_time_emb(orig.clone(), ts, inv_freq, W, T, window_duration, max_len)
    ref = _rotary_time_ref(orig, ts, inv_freq, W, T, window_duration, max_len)
    assert torch.equal(x[:, 4 * n_freq:], orig[:, 4 * n_freq:])
    assert not torch.equal(x[:, : 4 * n_freq], orig[:, : 4 * n_freq])
    _close(x, ref, 1e-5, "rotary time")
    _exact(x, ref, 0.9999, "rotary time")  # H100: 1.0


# ---------------------------------------------------------------------------------------------------- dispatch
_OURS = (r"\b(rmsnorm_rowblock_kernel|rmsnorm_kernel|layernorm_kernel|rope_kv_append_kernel|scatter_index_kernel|embed_scatter_kernel|"
         r"argmax_partial_kernel|argmax_final_kernel|im2col_conv1_kernel|im2col_conv2_kernel|pack_gate_up_kernel|logmel_init_max|"
         r"logmel_kernel|logmel_finalize|rotary_time_kernel)\b")


def _dispatch(ops):
    """(names of this file's kernels launched by one call per case, in launch order; the kernel each launch should be)."""
    calls, want = [], []

    def case(fn, *kernels):
        calls.append(fn)
        want.extend(kernels)

    for rows in RMS_ROWS:
        for dim in RMS_DIMS:
            x, w = _rand((rows, dim), 1.0, 1), _rand((dim,), 1.0, 2)
            case(lambda x=x, w=w: ops.rmsnorm(x, w, 1e-6), _rmsnorm_path(rows, dim))
            case(lambda x=x, w=w, i=_row_idx(rows, 3): ops.rmsnorm(x, w, 1e-6, row_idx=i), _rmsnorm_path(rows, dim))
    for dim in LN_DIMS:
        x, g = _rand((333, dim), 1.0, 4), _rand((dim,), 1.0, 5)
        case(lambda x=x, g=g: ops.layernorm(x, g, g), _ln_path(False, dim))
    for T, dim in POOL_CASES:
        x, g = _rand((3 * T, dim), 1.0, 6), _rand((dim,), 1.0, 7)
        case(lambda x=x, g=g, T=T: ops.avgpool_layernorm(x, 3, T, g, g), _ln_path(True, dim))
    for B, T, Tmax, pos0, starts, head_par in ROPE_CASES:
        qkv = _rand((B * T, 36 * 128), 1.0, 8)
        kv_start = torch.tensor(starts, dtype=torch.int32, device="cuda") if starts is not None else None
        case(lambda a=(qkv, B, T, 28, 4, 128, Tmax, pos0, kv_start): _rope_run(ops, *a),
             _tmpl("rope_kv_append_kernel", "true" if head_par else "false"))
    for n_tok, runs in SCATTER_CASES + [(3000, [(900, 1100), (1900, 2400)])]:
        case(lambda n=n_tok, r=runs: _scatter_case(ops, n, r, 9), "scatter_index_kernel", "embed_scatter_kernel")
    for V in ARGMAX_V:
        for B in ARGMAX_B:
            x = _rand((B, V), 1.0, 10, torch.float32)
            case(lambda x=x: ops.argmax(x), "argmax_partial_kernel", "argmax_final_kernel")
    for T in CONV1_T:
        x = _rand((2, 128, T), 1.0, 11, torch.float32)
        case(lambda x=x: ops.im2col_conv1(x), _tmpl("im2col_conv1_kernel", "float"))
        case(lambda x=x.to(bf16): ops.im2col_conv1(x), _tmpl("im2col_conv1_kernel", "__nv_bfloat16"))
    for T in CONV2_T:
        h = _rand((3 * T, 64), 1.0, 12)
        case(lambda h=h, T=T: ops.im2col_conv2(h, 3, T), "im2col_conv2_kernel")
    for F in (200, 18944):
        gu = _rand((F, 256), 1.0, 13)
        case(lambda gu=gu: ops.pack_gate_up(gu, gu), "pack_gate_up_kernel")
    tables = ops.LogMelTables(_mel_filters(), "cuda")
    wave = _rand((5, 80000), 0.1, 14, torch.float32)
    case(lambda: ops.logmel(wave, tables), "logmel_init_max", "logmel_kernel", "logmel_finalize")
    x, ts, inv = _rand((900, 64), 1.0, 15), torch.rand((3, 300), device="cuda") * 30, torch.rand((12,), device="cuda")
    case(lambda: ops.rotary_time_emb(x, ts, inv, 3, 300, 12.0, 1200), "rotary_time_kernel")

    return [n for n in _kernels(lambda: [fn() for fn in calls]) if re.search(_OURS, n)], want


def test_dispatch():
    """The kernel every case above runs, at the cases' shapes (contents do not steer the dispatch), in launch order.  The profiler
    session runs in a child process: CUPTI state left behind by a session can empty the next session of a later test."""
    root = Path(__file__).resolve().parents[1]
    code = (f"import json, sys; sys.path[:0] = [{str(root)!r}, {str(root / 'tests')!r}]; import test_cuda_core_kernels_gpu as m; "
            "from audio_flamingo_b200 import ops; print(json.dumps(m._dispatch(ops)))")
    r = subprocess.run([sys.executable, "-s", "-B", "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    ran, want = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(ran) == len(want), f"{len(ran)} launches of these kernels, {len(want)} expected: {ran}"
    for i, (name, kernel) in enumerate(zip(ran, want)):
        assert re.search(r"\b" + kernel + (r"\b" if "<" not in kernel else ""), name), f"launch {i}: {name}, expected {kernel}"
