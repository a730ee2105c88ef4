"""Torch-tensor front ends of the C-ABI kernels (one function per entry point of include/af3b200.h).

These only validate shapes/dtypes, allocate outputs with torch and pass raw pointers + the current CUDA stream
through ctypes.  All arithmetic happens in libaf3b200.so; nothing here falls back to torch ops.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib
from ._lib import EPI_BIAS, EPI_F32OUT, EPI_GELU, EPI_RESID, EPI_SWIGLU, EPI_SWIGLU_CONCAT, check, ptr, stream_ptr

bf16 = torch.bfloat16

# ---- instrumentation used by bench.py (counts are claims about OUR kernels; see DESIGN.md "measurement")
LAUNCHES = 0      # CUDA kernels launched through the C ABI since the last reset (graph replays add their captured count)
PROFILE = None    # when a dict: (kind, n_tok, n_feat, K, flags) -> list of (cuda start event, end event)
PHASE = None      # tag added to PROFILE keys ("decode" inside the cached decode step): bench.py weights those by the graph replays
TRACE_LOG = None  # when a list (af3_trace_begin open): (key, first slot, slot after the last) per C-ABI call, in launch order


def _count(n: int) -> None:
    global LAUNCHES
    LAUNCHES += n


class _Timed:
    """Brackets one C-ABI call with CUDA events on the current stream when PROFILE is enabled."""

    def __init__(self, key):
        self.key = key + (PHASE,) if PROFILE is not None else None
        self.tkey = key if TRACE_LOG is not None else None

    def __enter__(self):
        if self.tkey is not None:
            self.seq0 = _lib.load().af3_trace_seq()
        if self.key is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if self.tkey is not None:
            TRACE_LOG.append((self.tkey, self.seq0, _lib.load().af3_trace_seq()))
        if self.key is not None:
            self.e1.record()
            PROFILE.setdefault(self.key, []).append((self.e0, self.e1))
        return False


def _req(t: torch.Tensor, dtype, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.AF3Error(f"{name} must be a CUDA tensor (the AF3 hot path has no CPU fallback)")
    if t.dtype != dtype:
        raise _lib.AF3Error(f"{name} must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise _lib.AF3Error(f"{name} must be contiguous")
    if t.device.index != torch.cuda.current_device():
        # the C ABI launches on the current device (include/af3b200.h); launching cuda:0 kernels on cuda:1 pointers would fault
        raise _lib.AF3Error(f"{name} lives on {t.device} but the current CUDA device is cuda:{torch.cuda.current_device()}: "
                            "wrap the call in `with torch.cuda.device(...)` (the model's forward/generate do)")
    return t


# ----------------------------------------------------------------------------------------------- GEMM
_WORKSPACES = {}


def gemm_workspace(device):
    """Zero-initialised split-K workspace, one per device (GEMMs on a stream are serialised, so it is shared)."""
    key = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
    ws = _WORKSPACES.get(key)
    if ws is None:
        ws = torch.zeros((_lib.load().af3_gemm_workspace_bytes(),), device=torch.device("cuda", key), dtype=torch.uint8)
        _WORKSPACES[key] = ws
    return ws


def linear(x, w, bias=None, *, gelu=False, resid=None, res_period=0, out=None, out_f32=False):
    """out = epi(x @ w.T); x [n_tok, K] bf16, w [n_feat, K] bf16 (nn.Linear layout)."""
    lib = _lib.load()
    _req(x, bf16, "x"), _req(w, bf16, "w")
    n_tok, K = x.shape
    n_feat = w.shape[0]
    flags = 0
    if bias is not None:
        _req(bias, bf16, "bias")
        flags |= EPI_BIAS
    if gelu:
        flags |= EPI_GELU
    if resid is not None:
        _req(resid, bf16, "resid")
        flags |= EPI_RESID
    if out_f32:
        flags |= EPI_F32OUT
    if out is None:
        out = torch.empty((n_tok, n_feat), device=x.device, dtype=torch.float32 if out_f32 else bf16)
    ws = gemm_workspace(x.device) if n_tok <= 64 else None
    with _Timed(("gemm", n_tok, n_feat, K, flags)):
        check(
            lib.af3_gemm_bf16_ws(stream_ptr(), ptr(x), x.stride(0), ptr(w), w.stride(0), ptr(out), out.stride(0), n_tok, n_feat,
                                 K, flags, ptr(bias), ptr(resid), resid.stride(0) if resid is not None else 0, res_period,
                                 ptr(ws), ws.numel() if ws is not None else 0),
            "af3_gemm_bf16",
        )
    _count(1)
    return out


def lm_head_xent(x, w, labels, ignore_index=-100, *, store_logits=False):
    """LM head with ForCausalLMLoss's cross-entropy in its epilogue (include/af3b200.h af3_lm_head_xent).  x [n_tok, K] bf16,
    w [V, K] bf16, labels int64 [n_tok] already shifted.  -> (fp32 logits [n_tok, V] when store_logits else None, token_nll
    fp32 [n_tok] (0 where uncounted), totals fp64 [3] = {sum of nll, counted positions, invalid labels})."""
    lib = _lib.load()
    _req(x, bf16, "x"), _req(w, bf16, "w"), _req(labels, torch.int64, "labels")
    n_tok, K = x.shape
    V = w.shape[0]
    if labels.numel() != n_tok:
        raise _lib.AF3Error(f"lm_head_xent: labels must hold one label per token ({n_tok}), got {labels.numel()}")
    logits = torch.empty((n_tok, V), device=x.device, dtype=torch.float32) if store_logits else None
    token_nll = torch.empty((n_tok,), device=x.device, dtype=torch.float32)
    totals = torch.empty((3,), device=x.device, dtype=torch.float64)
    scratch = torch.empty((lib.af3_lm_head_xent_scratch_bytes(n_tok, V),), device=x.device, dtype=torch.uint8)
    with _Timed(("lm_head_xent", n_tok, V, K, int(store_logits))):
        check(lib.af3_lm_head_xent(stream_ptr(), ptr(x), x.stride(0), ptr(w), w.stride(0), n_tok, V, K, ptr(labels), int(ignore_index),
                                   ptr(logits), logits.stride(0) if logits is not None else 0, ptr(token_nll), ptr(totals), ptr(scratch)),
              "af3_lm_head_xent")
    _count(3)
    return logits, token_nll, totals


def pack_gate_up(gate, up):
    lib = _lib.load()
    _req(gate, bf16, "gate"), _req(up, bf16, "up")
    F, K = gate.shape
    packed = torch.empty((2 * ((F + 127) // 128) * 128, K), device=gate.device, dtype=bf16)
    check(lib.af3_pack_gate_up(stream_ptr(), ptr(gate), ptr(up), ptr(packed), F, K), "af3_pack_gate_up")
    _count(1)
    return packed


def swiglu_linear(x, w_packed, n_feat, out=None, concat=False):
    """out = silu(x @ gate.T) * (x @ up.T).  w_packed: from pack_gate_up (128-row interleave), or with concat=True the plain
    [gate; up] concatenation (n_feat % 128 == 0)."""
    lib = _lib.load()
    _req(x, bf16, "x"), _req(w_packed, bf16, "w_packed")
    n_tok, K = x.shape
    if out is None:
        out = torch.empty((n_tok, n_feat), device=x.device, dtype=bf16)
    with _Timed(("gemm", n_tok, n_feat, K, EPI_SWIGLU)):
        check(
            lib.af3_gemm_bf16_ws(stream_ptr(), ptr(x), x.stride(0), ptr(w_packed), w_packed.stride(0), ptr(out), out.stride(0),
                                 n_tok, n_feat, K, EPI_SWIGLU | (EPI_SWIGLU_CONCAT if concat else 0), None, None, 0, 0, None, 0),
            "af3_gemm_bf16(swiglu)",
        )
    _count(1)
    return out


# ----------------------------------------------------------------------------------------------- FP8 decoder projections
fp8 = torch.float8_e4m3fn


def quant_fp8(x, out=None, scales=None):
    """Dynamic 1 x 128 activation quantization (include/af3b200.h af3_quant_fp8).  x bf16 [rows, K], unit column stride (the
    row pitch may exceed K) -> (q float8_e4m3fn [rows, K], scales fp32 [K / 128, rows])."""
    lib = _lib.load()
    if not x.is_cuda or x.dtype != bf16 or x.dim() != 2 or x.stride(1) != 1:
        raise _lib.AF3Error("quant_fp8: x must be a CUDA bf16 [rows, K] tensor with unit column stride")
    rows, K = x.shape
    if out is None:
        out = torch.empty((rows, K), device=x.device, dtype=fp8)
    if scales is None:
        scales = torch.empty((K // 128, rows), device=x.device, dtype=torch.float32)
    # the kernel writes q with pitch K and the scales as [K / 128][rows]: caller buffers must have exactly that layout
    _req(out, fp8, "out"), _req(scales, torch.float32, "scales")
    if tuple(out.shape) != (rows, K) or tuple(scales.shape) != (K // 128, rows):
        raise _lib.AF3Error(f"quant_fp8: out must be [{rows}, {K}] and scales [{K // 128}, {rows}], got {tuple(out.shape)} and {tuple(scales.shape)}")
    with _Timed(("quant_fp8", rows, K, 0, 0)):
        check(lib.af3_quant_fp8(stream_ptr(), ptr(x), x.stride(0), ptr(out), ptr(scales), rows, K), "af3_quant_fp8")
    _count(1)
    return out, scales


def _fp8_operands(xq, w, w_scale_inv):
    q, sx = xq
    _req(q, fp8, "x"), _req(sx, torch.float32, "x_scales"), _req(w, fp8, "w"), _req(w_scale_inv, torch.float32, "w_scale_inv")
    n_tok, K = q.shape
    if tuple(sx.shape) != (K // 128, n_tok) or tuple(w_scale_inv.shape) != (w.shape[0] // 128, K // 128) or w.shape[1] != K:
        raise _lib.AF3Error(f"fp8 GEMM: shapes x {tuple(q.shape)}, x_scales {tuple(sx.shape)}, w {tuple(w.shape)}, "
                            f"w_scale_inv {tuple(w_scale_inv.shape)} do not match")
    return q, sx, n_tok, K


def linear_fp8(xq, w, w_scale_inv, bias=None, *, resid=None, out=None):
    """FP8Linear with 128 x 128 weight blocks: out = bf16(x @ w.T, block-scaled) [+ bias, rounded again] [+ resid].
    xq = quant_fp8(x); w float8_e4m3fn [n_feat, K]; w_scale_inv fp32 [n_feat / 128, K / 128]."""
    lib = _lib.load()
    q, sx, n_tok, K = _fp8_operands(xq, w, w_scale_inv)
    n_feat = w.shape[0]
    flags = 0
    if bias is not None:
        _req(bias, bf16, "bias")
        flags |= EPI_BIAS
    if resid is not None:
        _req(resid, bf16, "resid")
        flags |= EPI_RESID
    if out is None:
        out = torch.empty((n_tok, n_feat), device=q.device, dtype=bf16)
    ws = gemm_workspace(q.device) if n_tok <= 64 else None
    with _Timed(("gemm_fp8", n_tok, n_feat, K, flags)):
        check(
            lib.af3_gemm_fp8(stream_ptr(), ptr(q), q.stride(0), ptr(sx), ptr(w), w.stride(0), ptr(w_scale_inv), ptr(out), out.stride(0),
                             n_tok, n_feat, K, flags, ptr(bias), ptr(resid), resid.stride(0) if resid is not None else 0,
                             ptr(ws), ws.numel() if ws is not None else 0),
            "af3_gemm_fp8",
        )
    _count(1)
    return out


def swiglu_linear_fp8(xq, w_gate_up, w_scale_inv, n_feat, out=None):
    """out = silu(bf16(x @ gate.T)) * bf16(x @ up.T) with FP8 weights: w_gate_up the [gate; up] concatenation
    [2 n_feat, K], w_scale_inv its [2 n_feat / 128, K / 128] block scales."""
    lib = _lib.load()
    q, sx, n_tok, K = _fp8_operands(xq, w_gate_up, w_scale_inv)
    if w_gate_up.shape[0] != 2 * n_feat:
        raise _lib.AF3Error("swiglu_linear_fp8: w_gate_up must hold 2 * n_feat rows")
    if out is None:
        out = torch.empty((n_tok, n_feat), device=q.device, dtype=bf16)
    with _Timed(("gemm_fp8", n_tok, n_feat, K, EPI_SWIGLU)):
        check(
            lib.af3_gemm_fp8(stream_ptr(), ptr(q), q.stride(0), ptr(sx), ptr(w_gate_up), w_gate_up.stride(0), ptr(w_scale_inv), ptr(out),
                             out.stride(0), n_tok, n_feat, K, EPI_SWIGLU | EPI_SWIGLU_CONCAT, None, None, 0, None, 0),
            "af3_gemm_fp8(swiglu)",
        )
    _count(1)
    return out


def qkv_rope_linear_fp8(xq, w, w_scale_inv, bias, k_cache, v_cache, *, H, Hkv, D, rope_cs, pos_dev, out=None):
    """FP8 counterpart of qkv_rope_linear (few-token decode step): returns the [n_tok, (H+2Hkv)*D] buffer whose first H*D
    columns hold the rotated queries; rotated keys and the values go straight into the caches."""
    lib = _lib.load()
    q, sx, n_tok, K = _fp8_operands(xq, w, w_scale_inv)
    _req(bias, bf16, "bias")
    if out is None:
        out = torch.empty((n_tok, (H + 2 * Hkv) * D), device=q.device, dtype=bf16)
    ws = gemm_workspace(q.device)
    Tmax = k_cache.shape[2]
    with _Timed(("gemm_fp8", n_tok, (H + 2 * Hkv) * D, K, EPI_BIAS | 32)):
        check(
            lib.af3_gemm_qkv_rope_fp8(stream_ptr(), ptr(q), q.stride(0), ptr(sx), ptr(w), w.stride(0), ptr(w_scale_inv), ptr(bias), ptr(out),
                                      out.stride(0), n_tok, K, H, Hkv, D, ptr(rope_cs), ptr(k_cache), ptr(v_cache), Tmax, ptr(pos_dev),
                                      ptr(ws), ws.numel()),
            "af3_gemm_qkv_rope_fp8",
        )
    _count(1)
    return out


# ----------------------------------------------------------------------------------------------- log-mel
class LogMelTables:
    """Constant tables of the log-mel kernel, built exactly as the reference builds its constants."""

    def __init__(self, mel_filters_np: np.ndarray, device):
        # mel_filters_np: [201, 128] float64/32 from transformers.audio_utils.mel_filter_bank (WFE:95-103)
        f = np.asarray(mel_filters_np, dtype=np.float32)
        assert f.shape == (201, 128)
        nz = f != 0
        klo = np.where(nz.any(0), nz.argmax(0), 0).astype(np.int32)
        khi = np.where(nz.any(0), 200 - nz[::-1].argmax(0), -1).astype(np.int32)
        n = np.arange(201, dtype=np.float64)[:, None]
        k = np.arange(128, dtype=np.float64)[None, :]
        ang = 2.0 * np.pi * n * k / 400.0
        tab = np.stack([np.cos(ang), np.sin(ang)], axis=-1)
        tab[:, 101:, :] = 0.0
        self.filters = torch.from_numpy(f).to(device)
        self.klo = torch.from_numpy(klo).to(device)
        self.khi = torch.from_numpy(khi).to(device)
        self.table = torch.from_numpy(tab.astype(np.float32)).to(device).contiguous()
        self.hann = torch.hann_window(400, dtype=torch.float32).to(device)  # WFE:141


def logmel(wave, tables: LogMelTables):
    """wave fp32 [n_win, n_samples] -> fp32 [n_win, 128, n_samples // 160]  (WFE:135-164)."""
    lib = _lib.load()
    _req(wave, torch.float32, "wave")
    n_win, n_samples = wave.shape
    out = torch.empty((n_win, 128, n_samples // 160), device=wave.device, dtype=torch.float32)
    scratch = torch.empty((n_win,), device=wave.device, dtype=torch.int32)
    with _Timed(("logmel", n_win, n_samples, 0, 0)):
        check(
            lib.af3_logmel(stream_ptr(), ptr(wave), n_win, n_samples, ptr(tables.hann), ptr(tables.table), ptr(tables.filters),
                           ptr(tables.klo), ptr(tables.khi), ptr(out), ptr(scratch)),
            "af3_logmel",
        )
    _count(3)
    return out


# ----------------------------------------------------------------------------------------------- conv stem
def im2col_conv1(x):
    """x [n_win, C, T] fp32|bf16 -> [n_win*T, 3C] bf16."""
    lib = _lib.load()
    if x.dtype not in (torch.float32, bf16):
        raise _lib.AF3Error("input_features must be fp32 or bf16")
    _req(x, x.dtype, "input_features")
    n_win, Cc, T = x.shape
    cols = torch.empty((n_win * T, 3 * Cc), device=x.device, dtype=bf16)
    check(lib.af3_im2col_conv1(stream_ptr(), ptr(x), int(x.dtype == torch.float32), ptr(cols), n_win, Cc, T), "af3_im2col_conv1")
    _count(1)
    return cols


def im2col_conv2(h, n_win, T):
    """h [n_win*T, C] bf16 channel-last -> [n_win*T_out, 3C] bf16 (stride 2)."""
    lib = _lib.load()
    _req(h, bf16, "h")
    Cc = h.shape[1]
    T_out = (T - 1) // 2 + 1
    cols = torch.empty((n_win * T_out, 3 * Cc), device=h.device, dtype=bf16)
    check(lib.af3_im2col_conv2(stream_ptr(), ptr(h), ptr(cols), n_win, Cc, T), "af3_im2col_conv2")
    _count(1)
    return cols


# ----------------------------------------------------------------------------------------------- norms
def layernorm(x, gamma, beta, eps=1e-5, out=None):
    lib = _lib.load()
    _req(x, bf16, "x")
    rows, dim = x.shape
    if out is None:
        out = torch.empty_like(x)
    with _Timed(("layernorm", rows, dim, 0, 0)):
        check(lib.af3_layernorm(stream_ptr(), ptr(x), ptr(out), ptr(gamma), ptr(beta), rows, dim, eps), "af3_layernorm")
    _count(1)
    return out


def avgpool_layernorm(x, n_win, T, gamma, beta, eps=1e-5):
    lib = _lib.load()
    _req(x, bf16, "x")
    dim = x.shape[1]
    out = torch.empty((n_win * (T // 2), dim), device=x.device, dtype=bf16)
    with _Timed(("layernorm", n_win * (T // 2), dim, 0, 1)):
        check(lib.af3_avgpool_layernorm(stream_ptr(), ptr(x), ptr(out), ptr(gamma), ptr(beta), n_win, T, dim, eps), "af3_avgpool_layernorm")
    _count(1)
    return out


def rmsnorm(x, weight, eps=1e-6, row_idx=None, out=None):
    lib = _lib.load()
    _req(x, bf16, "x")
    dim = x.shape[1]
    rows = x.shape[0] if row_idx is None else row_idx.numel()
    if out is None:
        out = torch.empty((rows, dim), device=x.device, dtype=bf16)
    with _Timed(("rmsnorm", rows, dim, 0, 0)):
        check(lib.af3_rmsnorm(stream_ptr(), ptr(x), ptr(out), ptr(weight), rows, dim, eps, ptr(row_idx)), "af3_rmsnorm")
    _count(1)
    return out


# ----------------------------------------------------------------------------------------------- attention
def attention(q, k, v, out, *, B, H, Hkv, D, Tq, Tk, scale, causal, kv_layout=0, Tk_pitch=0, ldq=None, ldk=None,
              kv_len=None, kv_start=None):
    lib = _lib.load()
    with _Timed(("attention", B * H, Tq, Tk, D * 2 + int(causal))):
        check(
            lib.af3_attention(stream_ptr(), ptr(q), ldq, ptr(k), ptr(v), ldk, kv_layout, Tk_pitch, ptr(out), out.stride(-2),
                              B, H, Hkv, D, Tq, Tk, float(scale), int(causal), ptr(kv_len), ptr(kv_start)),
            "af3_attention",
        )
    _count(1)
    return out


def rope_kv_append(qkv, k_cache, v_cache, *, B, T, H, Hkv, D, pos0, inv_freq, kv_start=None, pos0_dev=None):
    lib = _lib.load()
    Tmax = k_cache.shape[2]
    with _Timed(("rope", B * T, H + 2 * Hkv, D, 0)):
        check(
            lib.af3_rope_kv_append(stream_ptr(), ptr(qkv), ptr(k_cache), ptr(v_cache), B, T, H, Hkv, D, Tmax, pos0, ptr(pos0_dev),
                                   ptr(kv_start), ptr(inv_freq)),
            "af3_rope_kv_append",
        )
    _count(1)


def rotary_time_emb(x, timestamps, inv_freq, W, T, window_duration, max_len):
    """Music Flamingo rotary time embedding, in place on x [W*T, dim] bf16."""
    lib = _lib.load()
    _req(x, bf16, "x"), _req(timestamps, torch.float32, "timestamps"), _req(inv_freq, torch.float32, "inv_freq")
    with _Timed(("rotary_time", W * T, x.shape[1], 0, 0)):
        check(lib.af3_rotary_time_emb(stream_ptr(), ptr(x), ptr(timestamps), ptr(inv_freq), W, T, x.shape[1], inv_freq.numel(),
                                      float(window_duration), float(max_len)), "af3_rotary_time_emb")
    _count(1)
    return x


def gated_residual(resid, y, alpha, row_gate=None, out=None):
    """out = resid + tanh(alpha) * y (Flamingo gate; alpha bf16 [dim] or 1 element); rows with row_gate == 0 take y = 0."""
    lib = _lib.load()
    _req(resid, bf16, "resid"), _req(y, bf16, "y"), _req(alpha, bf16, "alpha")
    rows, dim = resid.shape
    if out is None:
        out = torch.empty_like(resid)
    if row_gate is not None:
        _req(row_gate, torch.int32, "row_gate")
    with _Timed(("gated_residual", rows, dim, 0, 0)):
        check(lib.af3_gated_residual(stream_ptr(), ptr(resid), ptr(y), ptr(alpha), int(alpha.numel() == 1), ptr(row_gate), ptr(out), rows, dim),
              "af3_gated_residual")
    _count(1)
    return out


def rope_table(B, D, pos_dev, kv_start, inv_freq, out=None):
    """(cos, sin) of this decode step for every sequence: fp32 [B, D/2, 2] (shared by all layers)."""
    lib = _lib.load()
    if out is None:
        out = torch.empty((B, D // 2, 2), device=inv_freq.device, dtype=torch.float32)
    with _Timed(("rope_table", B, D, 0, 0)):
        check(lib.af3_rope_table(stream_ptr(), ptr(out), B, D, ptr(pos_dev), ptr(kv_start), ptr(inv_freq)), "af3_rope_table")
    _count(1)
    return out


def qkv_rope_linear(x, w, bias, k_cache, v_cache, *, H, Hkv, D, rope_cs, pos_dev, out=None):
    """Decode-step q/k/v projection with RoPE + KV append fused into the GEMM epilogue.  Returns the [n_tok, (H+2Hkv)*D]
    buffer whose first H*D columns hold the rotated queries (k / v go straight into the caches)."""
    lib = _lib.load()
    _req(x, bf16, "x"), _req(w, bf16, "w"), _req(bias, bf16, "bias")
    n_tok, K = x.shape
    if out is None:
        out = torch.empty((n_tok, (H + 2 * Hkv) * D), device=x.device, dtype=bf16)
    ws = gemm_workspace(x.device)
    Tmax = k_cache.shape[2]
    with _Timed(("gemm", n_tok, (H + 2 * Hkv) * D, K, EPI_BIAS | 32)):
        check(
            lib.af3_gemm_qkv_rope(stream_ptr(), ptr(x), x.stride(0), ptr(w), w.stride(0), ptr(bias), ptr(out), out.stride(0), n_tok, K,
                                  H, Hkv, D, ptr(rope_cs), ptr(k_cache), ptr(v_cache), Tmax, ptr(pos_dev), ptr(ws), ws.numel()),
            "af3_gemm_qkv_rope",
        )
    _count(1)
    return out


def decode_attention(qkv, k_cache, v_cache, out, scratch, *, B, H, Hkv, D, ctx_len, kv_start, scale):
    lib = _lib.load()
    Tmax = k_cache.shape[2]
    with _Timed(("decode_attention", B, H, Tmax, 0)):
        check(
            lib.af3_decode_attention(stream_ptr(), ptr(qkv), ptr(k_cache), ptr(v_cache), ptr(out), ptr(scratch), B, H, Hkv, D,
                                     Tmax, ptr(ctx_len), ptr(kv_start), float(scale)),
            "af3_decode_attention",
        )
    _count(1)
    return out


def decode_attention_scratch(B, H, D, Tmax, device):
    n = _lib.load().af3_decode_attention_scratch_bytes(B, H, D, Tmax)
    return torch.zeros(((n + 3) // 4,), device=device, dtype=torch.float32)  # zero: holds the arrival counters


# ----------------------------------------------------------------------------------------------- glue
def embed_scatter(ids, table, audio_token_id, audio_embeds, n_win, frames, post_len, out=None):
    """ids int64 [n_tok]; returns (inputs_embeds [n_tok, dim] bf16, counts int32[2] on device)."""
    lib = _lib.load()
    _req(ids, torch.int64, "input_ids"), _req(table, bf16, "embed_tokens.weight")
    n_tok = ids.numel()
    dim = table.shape[1]
    if out is None:
        out = torch.empty((n_tok, dim), device=table.device, dtype=bf16)
    scratch = torch.empty((n_tok,), device=table.device, dtype=torch.int32)
    counts = torch.zeros((2,), device=table.device, dtype=torch.int32)
    if audio_embeds is None:
        audio_embeds = table  # never read: n_win = 0 -> no valid rows
        n_win, frames = 0, 1
        post_len = counts
    with _Timed(("embed_scatter", n_tok, dim, 0, 0)):
        check(
            lib.af3_embed_scatter(stream_ptr(), ptr(ids), n_tok, ptr(table), dim, int(audio_token_id), ptr(audio_embeds), n_win,
                                  frames, ptr(post_len), ptr(out), ptr(scratch), ptr(counts)),
            "af3_embed_scatter",
        )
    _count(2)
    return out, counts


def token_step(raw_ids, unfinished, eos_ids, ctl, tok_buf, gen_idx, ids_out, done_flags):
    """Device-side bookkeeping of one greedy token (include/af3b200.h af3_token_step)."""
    lib = _lib.load()
    _req(raw_ids, torch.int64, "raw_ids"), _req(tok_buf, torch.int64, "tok_buf"), _req(unfinished, torch.int32, "unfinished")
    B, cap = tok_buf.shape
    with _Timed(("token_step", B, cap, 0, 0)):
        check(lib.af3_token_step(stream_ptr(), ptr(raw_ids), B, ptr(unfinished), ptr(eos_ids), ptr(ctl), ptr(tok_buf), cap, ptr(gen_idx),
                                 ptr(ids_out), ptr(done_flags)), "af3_token_step")
    _count(1)


def argmax(logits, out=None):
    lib = _lib.load()
    _req(logits, torch.float32, "logits")
    B, V = logits.shape
    if out is None:
        out = torch.empty((B,), device=logits.device, dtype=torch.int64)
    scratch = torch.empty((lib.af3_argmax_scratch_bytes(B),), device=logits.device, dtype=torch.uint8)
    with _Timed(("argmax", B, V, 0, 0)):
        check(lib.af3_argmax(stream_ptr(), ptr(logits), B, V, ptr(out), ptr(scratch)), "af3_argmax")
    _count(2)
    return out


def logits_process_argmax(logits, prompt_ids, generated_ids, gen_idx, tables, static_add, cap, out=None, scores=None):
    """Greedy logits processors + argmax in one pass over the logits (include/af3b200.h af3_logits_process_argmax).
    logits fp32 [B, V]; prompt_ids / generated_ids int64 [B, ld] (history = prompt_ids[:, :S] + generated_ids[:, :gen_idx]);
    gen_idx int32 [1]; tables int32 and static_add fp32 [V] from logits_process.compile_processors; scores: optional fp32
    [B, V] that receives the processed rows."""
    lib = _lib.load()
    _req(logits, torch.float32, "logits"), _req(prompt_ids, torch.int64, "prompt_ids"), _req(generated_ids, torch.int64, "generated_ids")
    _req(gen_idx, torch.int32, "gen_idx"), _req(tables, torch.int32, "tables"), _req(static_add, torch.float32, "static_add")
    B, V = logits.shape
    ld = prompt_ids.shape[1]
    if generated_ids.shape != prompt_ids.shape or prompt_ids.shape[0] != B or static_add.numel() != V:
        raise _lib.AF3Error("logits_process_argmax: prompt_ids / generated_ids must be [B, ld] and static_add [V]")
    if scores is not None:
        _req(scores, torch.float32, "scores")
        if tuple(scores.shape) != (B, V):
            raise _lib.AF3Error("logits_process_argmax: scores must be [B, V]")
    if out is None:
        out = torch.empty((B,), device=logits.device, dtype=torch.int64)
    scratch = torch.empty((lib.af3_logits_process_scratch_bytes(B, cap),), device=logits.device, dtype=torch.uint8)
    with _Timed(("logits_process", B, V, cap, int(scores is not None))):
        check(lib.af3_logits_process_argmax(stream_ptr(), ptr(logits), B, V, ptr(prompt_ids), ptr(generated_ids), ld, ptr(gen_idx), ptr(tables),
                                            ptr(static_add), cap, ptr(scores), ptr(out), ptr(scratch)), "af3_logits_process_argmax")
    _count(3)
    return out
