"""Both attention kernels against the restatements of oracle/attention_oracle.py, at every mask edge, row tiling and split.

attention_kernel<D, NWG> (attention_wgmma.cu) is called the way the product calls it: the encoder (kv_layout 0, D 64, the 1/8
folded into q, scale 1.0), the decoder prefill and its continuation chunks (kv_layout 1, causal GQA, left padding, a cache
pitch larger than Tk) and the cross-attention of xattn.py (K and V in one [B Tm, 2 H D] buffer).  decode_attn_kernel<8|16, 2>
(decode_attention.cu) runs with a split count the test knows: AF3_DECODE_SPLITS, or the host's rule for automatic cases.

Every case asserts three things about the kernel's bf16 output `out`:
  1. against the fp64 softmax `ref`, on every element:  |out - ref| <= 2^-8 (B + |ref|) (1 + slack) + 2^-126,
     B = sum p |v| / sum p.  The kernels round P to bf16 (relative error <= 2^-8 per weight) while the denominator sums the
     unrounded P, so the numerator is off by at most 2^-8 B; rounding the output to bf16 adds at most 2^-8 |out|.  slack covers
     the rest: every weight p_j = 2^(t_j - m) carries a relative error <= eps from the fp32 exponent t_j, and perturbing the
     weights by (1 + e_j), |e_j| <= eps, moves sum p v / sum p by at most eps (B + |ref|) / (1 - eps).  eps is bounded by
       - the fp32 score: q . k accumulated over D products in fp32, |error| <= 2 D 2^-24 A with A = max_j sum_d |q_d k_jd| scale
         (the factor 2 allows for the tensor core's truncating adds);
       - the fp32 scale * log2(e) and the fp32 rounding of t - m: <= 4 * 2^-24 A;
       - ex2.approx (<= 2^-22 relative) for p and for each rescale factor: (n_tiles + 2) 2^-22;
       - the fp32 accumulation of P . V and of the denominator over n_keys terms: 2 n_keys 2^-24;
     giving slack = 2^8 eps + 2^-7 (second order).  A grows with the peaked profiles (scores of hundreds of log units), so that is
     where slack matters.  A 1 % error in the softmax scale moves random rows by ~2 %, several times the bound.
  2. against the tile / split restatement: within one bf16 ulp (relative 2^-7) plus 2^-7 W, W = max_j (p_j / sum p) max_j |v_j|:
     where an fp32 score differs in its last bits, a P rounding can fall the other way and move the output by one bf16 ulp of
     that weight.  On an H100 a few elements per million need the W term (rows with few keys or one dominant key).
  3. a bit-identical fraction against the restatement of at least the floor below.  Differences come only from the fp32
     score accumulation order and ex2.approx landing next to a bf16 rounding tie of P or of the output.
     Lowest fraction over the cases, measured on an H100 80GB HBM3 (700 W): prefill 0.99636, decode 0.99634; floor 0.98 for
     both.  Summing the denominator from the bf16-rounded P instead of the fp32 P stays inside bounds 1 and 2 but drops the
     fraction to 0.91-0.94.

The prefill kernel must give identical bits with one and two consumer warpgroups per CTA (AF3_ATTN_V1=1 / default): both row
tilings run the same per-row arithmetic, and the extra tiles the wider tiling visits are fully masked for the other rows (alpha =
ex2.approx(0) = 1, p = +0, 0 * finite = +0).

Memory the kernels must not use holds poison: cache rows in [Tk, Tk_pitch) and rows past a kv_layout-0 buffer are NaN; keys
the kernel loads but masks (before kv_start, at or past kv_len / ctx) hold K = NaN or inf and V = 1e30.  The restatements see
clean copies.  The output buffer is wider than H D and longer than B Tq and its margins hold a sentinel.  Rows without a visible
key (causal rows before kv_start, kv_len = 0) must be exactly 0.

test_prefill and test_decode hold the new rows.  The rows of the older suite run through the same checks under their old names
in test_kernels_gpu.py (test_attention_bidirectional, test_attention_causal_gqa_cache,
test_attention_v2_matches_v1_on_a_live_cache_offset, test_decode_attention); their cases are listed here.
test_dispatch checks by torch.profiler kernel name which instantiation every case of both files runs (one session, in a child
process).
"""
import json
import math
import os
import re
import subprocess
import sys
import zlib
from pathlib import Path

import pytest
import torch

from oracle import attention_oracle as A

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
SENT = -7.5
DEV = "cuda"
PREFILL_FLOOR = 0.98
DECODE_FLOOR = 0.98


@pytest.fixture(scope="module")
def ops():
    from audio_flamingo_b200 import ops as _ops

    return _ops


def _rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(bf16).to(DEV)


def _poison_keys(k, v, j0, j1, inf):
    """K = NaN (or +inf), V = 1e30 on rows [j0, j1) of k / v [..., T, D] (masked keys the kernel loads)."""
    if j1 > j0:
        k[..., j0:j1, :] = math.inf if inf else math.nan
        v[..., j0:j1, :] = 1e30


# ---------------------------------------------------------------------------------------------------- prefill kernel
# (kind, B, H, Hkv, D, Tq, Tk, per-sequence kv_len (enc / x) or kv_start (dec), profile)
#   enc: encoder self-attention, kv_layout 0, Tq = Tk;  dec: decoder prefill / continuation, kv_layout 1, causal, pitch Tk + 200;
#   x: cross-attention, q [B Tq, H D], K / V in one [B Tk, 2 H D] buffer
PREFILL = [
    ("enc", 4, 20, 20, 64, 1500, 1500, [0, 1, 127, 128], "random"),
    ("enc", 4, 20, 20, 64, 1500, 1500, [129, 1499, 1500, 1600], "random"),
    ("enc", 4, 20, 20, 64, 1500, 1500, [1, 127, 128, 1499], "edges"),
    ("enc", 3, 3, 3, 64, 333, 333, [333, 100, 7], "random"),
    ("enc", 2, 2, 2, 128, 300, 300, [300, 1], "edges"),
    ("enc", 2, 4, 4, 64, 65, 65, None, "random"),
    ("dec", 7, 28, 4, 128, 780, 780, [0, 1, 127, 128, 129, 255, 779], "random"),
    ("dec", 7, 28, 4, 128, 780, 780, [0, 1, 127, 128, 129, 255, 779], "edges"),
    ("dec", 2, 28, 4, 128, 780, 780, [0, 3], "diagonal"),
    ("dec", 3, 28, 4, 128, 1000, 1000, [0, 3, 530], "rising"),
    ("dec", 3, 28, 4, 128, 1000, 1000, [0, 3, 530], "falling"),
    ("dec", 2, 28, 4, 128, 780, 780, None, "two_peaks"),
    ("dec", 2, 28, 4, 128, 1, 1, [0, 0], "random"),
    ("dec", 2, 28, 4, 128, 63, 63, [0, 62], "diagonal"),
    ("dec", 2, 28, 4, 128, 64, 64, [0, 1], "random"),
    ("dec", 2, 28, 4, 128, 65, 65, [0, 64], "diagonal"),
    ("dec", 2, 28, 4, 128, 127, 127, [0, 126], "edges"),
    ("dec", 2, 28, 4, 128, 128, 128, [0, 127], "diagonal"),
    ("dec", 2, 28, 4, 128, 129, 129, [0, 128], "edges"),
    ("dec", 2, 4, 4, 128, 300, 300, [0, 37], "diagonal"),        # GQA 1
    ("dec", 2, 8, 1, 128, 513, 513, [0, 400], "random"),        # GQA 8
    ("dec", 2, 8, 2, 128, 256, 256, None, "random"),
    ("dec", 2, 28, 4, 128, 1, 650, [0, 77], "edges"),           # continuation chunks: Tq new rows after Tk - Tq cached keys
    ("dec", 2, 28, 4, 128, 129, 385, [0, 130], "diagonal"),
    ("dec", 2, 28, 4, 128, 200, 650, [127, 255], "edges"),
    ("dec", 2, 8, 1, 128, 129, 300, [1, 128], "diagonal"),
    ("x", 2, 4, 4, 64, 37, 1, [1, 1], "random"),
    ("x", 2, 4, 4, 128, 37, 5, [5, 2], "random"),
    ("x", 2, 4, 4, 64, 37, 40, [40, 17], "edges"),
    ("x", 2, 4, 4, 128, 100, 127, [127, 126], "edges"),
    ("x", 2, 4, 4, 64, 37, 129, [129, 128], "edges"),
    ("x", 2, 4, 4, 128, 300, 1500, [1500, 1037], "random"),
]


def _prefill_case(c):
    """-> dict: kernel call arguments, clean oracle tensors, output buffer."""
    kind, B, H, Hkv, D, Tq, Tk, per_seq, profile = c
    seed = zlib.crc32(repr(c).encode()) % 1000
    scale = 1.0 if kind == "enc" else D ** -0.5
    HD = H * D
    kv_len = per_seq if kind in ("enc", "x") else None
    kv_start = per_seq if kind == "dec" else None
    r = dict(B=B, H=H, Hkv=Hkv, D=D, Tq=Tq, Tk=Tk, scale=scale, causal=kind == "dec", kv_len=kv_len, kv_start=kv_start)
    if kind == "enc":
        big = _rand((B * Tk + 256, 3 * HD), seed)
        big[:, :HD] = (big[:, :HD].float() * 0.125).to(bf16)            # the encoder folds 1/8 into q
        qkv = big[:B * Tk]
        q4 = qkv[:, :HD].view(B, Tq, H, D)
        k4 = qkv[:, HD:2 * HD].view(B, Tk, H, D).transpose(1, 2)
        v4 = qkv[:, 2 * HD:].view(B, Tk, H, D).transpose(1, 2)
        args = (qkv, qkv[:, HD:], qkv[:, 2 * HD:])
        kw = dict(kv_layout=0, ldq=3 * HD, ldk=3 * HD)
    elif kind == "x":
        q = _rand((B * Tq, HD), seed)
        big = _rand((B * Tk + 64, 2 * HD), seed + 1)
        kv = big[:B * Tk]
        q4 = q.view(B, Tq, H, D)
        k4 = kv[:, :HD].view(B, Tk, H, D).transpose(1, 2)
        v4 = kv[:, HD:].view(B, Tk, H, D).transpose(1, 2)
        args = (q, kv, kv[:, HD:])
        kw = dict(kv_layout=0, ldq=HD, ldk=2 * HD)
    else:
        pitch = Tk + 200
        qbuf = _rand((B * Tq, (H + 2 * Hkv) * D), seed)
        k4, v4 = _rand((B, Hkv, pitch, D), seed + 1), _rand((B, Hkv, pitch, D), seed + 2)
        q4 = qbuf.view(B, Tq, H + 2 * Hkv, D)[:, :, :H]
        args = (qbuf, k4, v4)
        kw = dict(kv_layout=1, Tk_pitch=pitch, ldq=(H + 2 * Hkv) * D, ldk=D)
        k4, v4 = k4[:, :, :Tk], v4[:, :, :Tk]
    lens = [min(n, Tk) for n in (kv_len or [Tk] * B)]
    starts = kv_start or [0] * B
    for b in range(B):
        if profile == "edges":
            for hk in range(Hkv):
                A.edge_probe(q4[b], k4[b, hk], v4[b, hk], scale, masked=[lens[b]] + ([starts[b] - 1] if kv_start else []),
                             visible=[lens[b] - 1] + ([starts[b]] if kv_start else []))
        elif profile == "diagonal":
            A.diagonal_probe(q4[b], k4[b].transpose(0, 1), scale, Tk - Tq)
        elif profile != "random":
            j = torch.arange(Tk, device=DEV, dtype=torch.float32)[:, None]
            first, last = starts[b] + Tk // 4, (Tk - 1 if profile == "rising" else 3 * Tk // 4)
            A.peak_scores(q4[b], k4[b].transpose(0, 1), profile, scale, first, last, j)
    r["clean"] = (q4.clone(), k4.clone(), v4.clone())
    # poison: masked keys the kernel loads, rows past Tk in the cache pitch, rows past a packed buffer
    for b in range(B):
        _poison_keys(k4[b], v4[b], 0, starts[b], b % 2)
        _poison_keys(k4[b], v4[b], lens[b], Tk, b % 2)
    if kind == "dec":
        args[1][:, :, Tk:] = math.nan
        args[2][:, :, Tk:] = math.nan
    else:
        big[B * Tk:] = math.nan
    out_big = torch.full((B * Tq + 5, HD + 64), SENT, device=DEV, dtype=bf16)
    ld = HD + 64     # as_strided: a view would give a Tq = 1 output any row stride, and ops.attention passes stride(-2) as ldo
    r.update(args=args, kw=kw, out_big=out_big, out=out_big.as_strided((B, Tq, HD), (Tq * ld, ld, 1)))
    return r


def _prefill_call(ops, r):
    kv_len = torch.tensor(r["kv_len"], dtype=torch.int32, device=DEV) if r["kv_len"] else None
    kv_start = torch.tensor(r["kv_start"], dtype=torch.int32, device=DEV) if r["kv_start"] else None
    ops.attention(*r["args"], r["out"], B=r["B"], H=r["H"], Hkv=r["Hkv"], D=r["D"], Tq=r["Tq"], Tk=r["Tk"], scale=r["scale"],
                  causal=r["causal"], kv_len=kv_len, kv_start=kv_start, **r["kw"])


def _check(out, clean_ref, rest, what, floor):
    """Assertions 1-3 of the module docstring.  out, rest: bf16; clean_ref: (ref, bnd, smag, wmax, D, n_keys)."""
    ref, bnd, smag, wmax, D, n_keys = clean_ref
    o = out.double()
    tol = A.attention_tolerance(ref, bnd, smag, D, n_keys)
    err = (o - ref).abs()
    bad = ~(err <= tol)
    assert not bad.any(), f"{what}: {int(bad.sum())}/{o.numel()} outside the fp64 bound, worst err / tol {(err / tol).max().item():.3g}"
    rd = rest.double()
    err = (o - rd).abs()
    bad = ~(err <= 2.0 ** -7 * (rd.abs() + wmax))
    assert not bad.any(), f"{what}: {int(bad.sum())}/{o.numel()} more than one bf16 ulp from the restatement"
    frac = (out == rest).double().mean().item()
    print(f"\n{what}: bit-identical fraction {frac:.6f}")
    assert frac >= floor, f"{what}: bit-identical fraction {frac:.6f} < {floor}"


# Rows of the older suite, kept under their names in test_kernels_gpu.py and run through check_prefill / check_decode.
# test_attention_bidirectional (D, H, T, kv_len): encoder layout, B = 3 with kv_len, else 2
BIDIRECTIONAL = [(64, 4, 200, None), (64, 20, 1500, None), (64, 3, 333, [333, 100, 7]), (128, 2, 256, None),
                 (64, 2, 1500, [1500, 385, 12]), (128, 3, 700, [700, 129, 256]), (64, 2, 65, None),
                 (128, 2, 300, [300, 1, 190]), (64, 5, 2000, [2000, 1999, 640])]
# test_attention_causal_gqa_cache (T, kv_start, profile): causal GQA 8:2, B = len(kv_start) or 2
CAUSAL = [(256, None, "random"), (300, [0, 37, 250], "random"), (130, [5, 129], "random"), (780, [0, 3, 530], "random"),
          (1000, None, "random"), (64, None, "random"), (129, [0, 128], "random"), (513, [0, 400, 512], "random"),
          (1000, [0, 3, 530], "rising"), (1000, [0, 3, 530], "falling"), (780, None, "two_peaks")]
# test_attention_v2_matches_v1_on_a_live_cache_offset: a continuation chunk, 200 new rows after 450 cached keys
CONTINUATION = ("dec", 2, 28, 4, 128, 200, 650, [0, 77], "random")


def bidirectional_case(D, H, T, lens):
    return ("enc", 3 if lens else 2, H, H, D, T, T, lens, "random")


def causal_case(T, starts, scores):
    return ("dec", len(starts) if starts else 2, 8, 2, 128, T, T, starts, scores)


def check_prefill(ops, monkeypatch, case):
    """Both row tilings give identical bits; the output meets assertions 1-3, leaves the margins alone and is 0 in rows
    without a visible key."""
    r = _prefill_case(case)
    outs = {}
    for v1 in ("1", "0"):
        monkeypatch.setenv("AF3_ATTN_V1", v1)
        r["out_big"].fill_(SENT)
        _prefill_call(ops, r)
        torch.cuda.synchronize()
        outs[v1] = r["out_big"].clone()
    assert torch.equal(outs["0"], outs["1"]), "one and two warpgroups per CTA must give identical bits"
    B, Tq, H, D, Tk = r["B"], r["Tq"], r["H"], r["D"], r["Tk"]
    ob = outs["0"]
    assert (ob[B * Tq:] == SENT).all() and (ob[:, H * D:] == SENT).all(), "write outside the output rows / columns"
    out = ob[:B * Tq, :H * D].reshape(B, Tq, H, D)
    q, k, v = r["clean"]
    a = (q, k, v, r["scale"], r["causal"], r["kv_len"], r["kv_start"])
    ref, bnd, smag, wmax = A.softmax_attention_fp64(*a)
    empty = ~A.visible_mask(B, Tq, Tk, r["causal"], r["kv_len"], r["kv_start"], DEV).any(-1)
    assert (out[empty] == 0).all(), "rows without a visible key must be 0"
    _check(out, (ref, bnd, smag, wmax, D, Tk), A.prefill_tile_restatement(*a), "prefill", PREFILL_FLOOR)


@pytest.mark.parametrize("case", PREFILL, ids=lambda c: "-".join(str(x) for x in c[:2] + c[5:7] + (c[8],)) + f"-H{c[2]}:{c[3]}-D{c[4]}")
def test_prefill(ops, monkeypatch, case):
    check_prefill(ops, monkeypatch, case)


# ---------------------------------------------------------------------------------------------------- decode kernel
# (B, H, Hkv, Tmax, ctx, kv_start per sequence, splits: int = AF3_DECODE_SPLITS, "auto" = the host's rule, profile)
DECODE = [
    (5, 28, 4, 1024, 257, [0, 1, 127, 128, 256], "auto", "random"),   # G 7; auto: 132 SMs / 20 = 6 splits over 1-3 live chunks
    (5, 28, 4, 1024, 257, [0, 1, 127, 128, 256], 1, "edges"),
    (2, 8, 2, 512, 1, [0, 0], 1, "random"),                          # a single key; G 4
    (2, 8, 2, 512, 1, [0, 0], 3, "edges"),                           # ... three splits, two idle
    (3, 10, 2, 512, 127, [0, 1, 126], 2, "edges"),                    # G 5
    (3, 14, 2, 512, 128, [0, 1, 127], 3, "random"),                   # G 7
    (4, 16, 2, 512, 129, [0, 1, 127, 128], "auto", "edges"),          # G 8: the widest NG = 8 group
    (3, 18, 2, 768, 255, [0, 128, 254], 2, "rising"),                 # G 9: the narrowest NG = 16 group
    (4, 24, 2, 768, 256, [0, 1, 127, 128], 5, "edges"),               # G 12, more splits than live chunks
    (4, 26, 2, 1024, 1024, [0, 1, 128, 1023], 99, "falling"),         # G 13, ctx = Tmax, split count clamped to chunks(Tmax)
    (3, 26, 2, 1024, 257, [0, 128, 256], 1, "edges"),
    (2, 32, 2, 2048, 1901, [5, 1300], 4, "two_peaks"),                # G 16: no padded head
    (2, 32, 2, 2048, 1901, [5, 1300], 1, "edges"),
    (2, 4, 4, 1024, 700, [0, 300], 3, "edges"),                       # G 1: seven padded heads of NG = 8
    (1, 28, 4, 4096, 3000, [0], "auto", "random"),                    # B = 1: auto gives 32 splits (clamped), 24 live
]


# test_decode_attention (B, H, Hkv, Tmax, ctx, kv_start, splits or None = the host's rule, profile), older rows
DECODE_PORTED = [
    (3, 28, 4, 1024, 777, [0, 100, 776], None, "random"),   # auto: one chunk per split
    (3, 28, 4, 1024, 777, [0, 100, 776], 1, "random"),      # one CTA streams 7 chunks (the ring wraps)
    (3, 28, 4, 1024, 777, [0, 100, 776], 3, "random"),      # 3 / 3 / 1 chunks; row 2 has a single live key
    (2, 16, 1, 2048, 1901, [5, 1300], 1, "random"),         # G = 16 (no padded heads), 15 chunks in one CTA
    (2, 8, 4, 2048, 1537, [0, 640], 5, "random"),           # G = 2, uneven splits, last chunk holds one key
    (40, 28, 4, 512, 300, None, None, "random"),            # B * Hkv > SM count -> nz = 1, more CTAs than SMs
    (1, 28, 4, 128, 1, [0], None, "random"),                # a single key
    (2, 4, 4, 1024, 700, [0, 300], None, "random"),         # G = 1: seven padded heads of NG = 8
    (2, 4, 4, 1024, 700, [0, 300], 3, "random"),
    (2, 32, 4, 1024, 700, [0, 300], None, "random"),        # G = 8: the widest NG = 8 group
    (2, 32, 4, 1024, 700, [0, 300], 3, "random"),
    (2, 36, 4, 1024, 700, [0, 300], None, "random"),        # G = 9: the narrowest NG = 16 group
    (2, 36, 4, 1024, 700, [0, 300], 3, "random"),
    (2, 28, 4, 2048, 1901, [0, 300], 1, "rising"),          # running max moves every chunk inside one CTA
    (2, 28, 4, 2048, 1901, [0, 300], None, "rising"),       # ... and across the split partials (one chunk each)
    (2, 28, 4, 2048, 1901, [0, 300], 3, "falling"),         # maximum in the first chunk
    (2, 28, 4, 2048, 1901, [5, 1300], 4, "two_peaks"),      # equal peaks in the first and the last split
]


def ported_decode_case(B, H, Hkv, Tmax, ctx, starts, splits, scores):
    return (B, H, Hkv, Tmax, ctx, starts, "auto" if splits is None else splits, scores)


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _decode_case(c):
    B, H, Hkv, Tmax, ctx, starts, splits, profile = c
    seed = zlib.crc32(repr(c).encode()) % 1000
    D, scale = 128, 128 ** -0.5
    qkv = _rand((B, (H + 2 * Hkv) * D), seed)
    kc, vc = _rand((B, Hkv, Tmax, D), seed + 1), _rand((B, Hkv, Tmax, D), seed + 2)
    st = starts or [0] * B
    q3 = qkv[:, :H * D].view(B, H, D)
    for b in range(B):
        if profile == "edges":
            for hk in range(Hkv):
                A.edge_probe(q3[b], kc[b, hk], vc[b, hk], scale, masked=[st[b] - 1, ctx], visible=[st[b], ctx - 1])
        elif profile != "random":
            first, last = st[b] + 3, ctx - 4
            if profile == "rising":
                last = ctx - 1
            A.peak_scores(q3[b], kc[b], profile, scale, first, last, torch.arange(Tmax, device=DEV, dtype=torch.float32)[None, :])
    clean = (q3.clone(), kc.clone(), vc.clone())
    for b in range(B):
        _poison_keys(kc[b], vc[b], 0, st[b], b % 2)
        _poison_keys(kc[b], vc[b], ctx, Tmax, b % 2)
    nz = A.decode_splits(B, Hkv, Tmax, _sm_count(), None if splits == "auto" else splits)
    return dict(B=B, H=H, Hkv=Hkv, D=D, Tmax=Tmax, ctx=ctx, starts=starts, splits=splits, nz=nz, scale=scale, qkv=qkv, kc=kc, vc=vc,
                clean=clean, ctx_len=torch.tensor([ctx], dtype=torch.int32, device=DEV),
                kv_start=torch.tensor(starts, dtype=torch.int32, device=DEV) if starts else None)


def _set_splits(splits):
    if splits == "auto":
        os.environ.pop("AF3_DECODE_SPLITS", None)
    else:
        os.environ["AF3_DECODE_SPLITS"] = str(splits)


def _decode_call(ops, r, out, scratch):
    ops.decode_attention(r["qkv"], r["kc"], r["vc"], out, scratch, B=r["B"], H=r["H"], Hkv=r["Hkv"], D=r["D"], ctx_len=r["ctx_len"],
                         kv_start=r["kv_start"], scale=r["scale"])


def _counters(scratch, B, H):
    """The split arrival counters: the last B H int32 words of the scratch."""
    return scratch.view(torch.int32)[-B * H:]


def _decode_refs(r):
    q, k, v = r["clean"]
    ctx = r["ctx"]
    ref, bnd, smag, wmax = A.softmax_attention_fp64(q[:, None], k[:, :, :ctx], v[:, :, :ctx], r["scale"], kv_start=r["starts"])
    rest = A.decode_split_restatement(q, k, v, r["scale"], ctx, r["starts"], r["nz"])
    return (ref[:, 0], bnd[:, 0], smag[:, 0], wmax[:, 0], r["D"], ctx), rest


def check_decode(ops, monkeypatch, case):
    """Assertions 1-3 at the case's split count; the margins of the output are untouched and the arrival counters zero."""
    monkeypatch.setenv("AF3_DECODE_SPLITS", "1")   # restored after the test
    r = _decode_case(case)
    B, H, D = r["B"], r["H"], r["D"]
    _set_splits(r["splits"])
    out = torch.full((B + 2, H * D), SENT, device=DEV, dtype=bf16)
    scratch = ops.decode_attention_scratch(B, H, D, r["Tmax"], DEV)
    _decode_call(ops, r, out[:B], scratch)
    torch.cuda.synchronize()
    assert (out[B:] == SENT).all()
    assert not _counters(scratch, B, H).any(), "split arrival counters must be left at zero"
    ref, rest = _decode_refs(r)
    _check(out[:B].view(B, H, D), ref, rest, f"decode nz={r['nz']}", DECODE_FLOOR)


@pytest.mark.parametrize("case", DECODE, ids=lambda c: f"B{c[0]}-H{c[1]}:{c[2]}-ctx{c[4]}-nz{c[6]}-{c[7]}")
def test_decode(ops, monkeypatch, case):
    check_decode(ops, monkeypatch, case)


@pytest.mark.parametrize("splits", [3, "auto"])
def test_decode_graph_replay_steps_ctx(ops, monkeypatch, splits):
    """One captured call, ctx_len stepped on the device across chunk edges: every replay equals an eager call at that ctx."""
    monkeypatch.setenv("AF3_DECODE_SPLITS", "1")
    r = _decode_case((3, 28, 4, 512, 130, [0, 1, 127], splits, "random"))
    _set_splits(splits)
    B, H, D = r["B"], r["H"], r["D"]
    out_g, out_e = torch.zeros((B, H * D), device=DEV, dtype=bf16), torch.zeros((B, H * D), device=DEV, dtype=bf16)
    scr_g = ops.decode_attention_scratch(B, H, D, r["Tmax"], DEV)
    scr_e = ops.decode_attention_scratch(B, H, D, r["Tmax"], DEV)
    # the replays read past the ctx the case poisoned from: use the clean cache
    r["kc"].copy_(r["clean"][1])
    r["vc"].copy_(r["clean"][2])
    ctx_g = torch.tensor([127], dtype=torch.int32, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.decode_attention(r["qkv"], r["kc"], r["vc"], out_g, scr_g, B=B, H=H, Hkv=r["Hkv"], D=D, ctx_len=ctx_g, kv_start=r["kv_start"],
                             scale=r["scale"])
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.decode_attention(r["qkv"], r["kc"], r["vc"], out_g, scr_g, B=B, H=H, Hkv=r["Hkv"], D=D, ctx_len=ctx_g, kv_start=r["kv_start"],
                             scale=r["scale"])
    for ctx in (127, 128, 129, 130, 255, 256, 257, 258):
        ctx_g.fill_(ctx)
        out_g.zero_()
        g.replay()
        r["ctx_len"].fill_(ctx)
        _decode_call(ops, r, out_e, scr_e)
        torch.cuda.synchronize()
        assert torch.equal(out_g, out_e), f"replay at ctx {ctx} differs from the eager call"
        assert not _counters(scr_g, B, H).any() and not _counters(scr_e, B, H).any()


def test_decode_reads_the_key_appended_just_before(ops, monkeypatch):
    """The decode step's chain: qkv_rope_linear appends the new key and value at slot ctx - 1, decode_attention reads them.  The
    older cache rows hold K = V = 0, so every bit of the output comes from the appended row: reading the slot before the
    producer has written it gives 0.  PDL on, PDL off and the unfused chain (GEMM, rope_kv_append, attention) agree bit for
    bit, and with the restatement."""
    from audio_flamingo_b200 import _lib

    monkeypatch.setenv("AF3_DECODE_SPLITS", "1")
    B, H, Hkv, D, K, Tmax, ctx = 4, 28, 4, 128, 512, 256, 130
    x, w, bias = _rand((B, K), 60), _rand(((H + 2 * Hkv) * D, K), 61, 0.05), _rand(((H + 2 * Hkv) * D,), 62, 0.3)
    inv_freq = (1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).cuda()
    pos = torch.tensor([ctx - 1], dtype=torch.int32, device=DEV)
    ctx_len = torch.tensor([ctx], dtype=torch.int32, device=DEV)
    starts = torch.tensor([0, 1, 127, 129], dtype=torch.int32, device=DEV)

    def chain(fused):
        kc = torch.zeros((B, Hkv, Tmax, D), device=DEV, dtype=bf16)
        vc = torch.zeros_like(kc)
        scratch = ops.decode_attention_scratch(B, H, D, Tmax, DEV)
        out = torch.zeros((B, H * D), device=DEV, dtype=bf16)
        if fused:
            cs = ops.rope_table(B, D, pos, starts, inv_freq)
            qkv = ops.qkv_rope_linear(x, w, bias, kc, vc, H=H, Hkv=Hkv, D=D, rope_cs=cs, pos_dev=pos)
        else:
            qkv = ops.linear(x, w, bias)
            ops.rope_kv_append(qkv, kc, vc, B=B, T=1, H=H, Hkv=Hkv, D=D, pos0=0, inv_freq=inv_freq, kv_start=starts, pos0_dev=pos)
        ops.decode_attention(qkv, kc, vc, out, scratch, B=B, H=H, Hkv=Hkv, D=D, ctx_len=ctx_len, kv_start=starts, scale=D ** -0.5)
        torch.cuda.synchronize()
        return out, qkv, kc, vc

    lib = _lib.load()
    try:
        lib.af3_set_pdl(1)
        on, qkv, kc, vc = chain(True)
    finally:
        lib.af3_set_pdl(0)
    off = chain(True)[0]
    unfused = chain(False)[0]
    assert torch.equal(on, off) and torch.equal(on, unfused)
    # every older row has K = V = 0, so each output element is a positive multiple of the appended value
    v_new = vc[:, :, ctx - 1].repeat_interleave(H // Hkv, dim=1).reshape(B, H * D).float()
    assert (v_new != 0).float().mean() > 0.99 and torch.equal(on.float().sign(), v_new.sign())
    r = dict(clean=(qkv[:, :H * D].view(B, H, D), kc, vc), ctx=ctx, scale=D ** -0.5, starts=starts.tolist(), nz=1, D=D)
    ref, rest = _decode_refs(r)
    _check(on.view(B, H, D), ref, rest, "decode after append", DECODE_FLOOR)


# ---------------------------------------------------------------------------------------------------- dispatch
def _dispatch(ops):
    """(names of the attention kernels launched by one call per case, in launch order; the kernel each should be)."""
    from test_cuda_core_kernels_gpu import _kernels, _tmpl

    calls, want = [], []
    prefill = PREFILL + [bidirectional_case(*c) for c in BIDIRECTIONAL] + [causal_case(*c) for c in CAUSAL] + [CONTINUATION]
    for c in prefill:
        r = _prefill_case(c)
        for v1 in ("1", "0"):
            calls.append(lambda r=r, v1=v1: (os.environ.__setitem__("AF3_ATTN_V1", v1), _prefill_call(ops, r)))
            want.append(_tmpl("attention_kernel", str(r["D"]), "1" if v1 == "1" else "2"))
    for c in DECODE + [ported_decode_case(*c) for c in DECODE_PORTED]:
        r = _decode_case(c)
        scratch = ops.decode_attention_scratch(r["B"], r["H"], r["D"], r["Tmax"], DEV)
        out = torch.empty((r["B"], r["H"] * r["D"]), device=DEV, dtype=bf16)
        calls.append(lambda r=r, s=scratch, o=out: (_set_splits(r["splits"]), _decode_call(ops, r, o, s)))
        want.append(_tmpl("decode_attn_kernel", "8" if r["H"] // r["Hkv"] <= 8 else "16", "2"))
    names = _kernels(lambda: [fn() for fn in calls])
    return [n for n in names if re.search(r"attention_kernel|decode_attn_kernel", n)], want


def test_dispatch():
    """The instantiation every case above runs: attention_kernel<D, NWG>, decode_attn_kernel<8|16, 2>.  The profiler session runs
    in a child process: CUPTI state left behind by a session can empty the next session of a later test."""
    root = Path(__file__).resolve().parents[1]
    code = (f"import json, sys; sys.path[:0] = [{str(root)!r}, {str(root / 'tests')!r}]; import test_attention_kernels_gpu as m; "
            "from audio_flamingo_b200 import ops; print(json.dumps(m._dispatch(ops)))")
    env = {k: v for k, v in os.environ.items() if k not in ("AF3_ATTN_V1", "AF3_DECODE_SPLITS")}
    r = subprocess.run([sys.executable, "-s", "-B", "-c", code], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    ran, want = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(ran) == len(want), f"{len(ran)} launches of the attention kernels, {len(want)} expected: {ran}"
    for i, (name, kernel) in enumerate(zip(ran, want)):
        assert re.search(r"\b" + kernel, name), f"launch {i}: {name}, expected {kernel}"
