"""ORACLE -- TEST INFRASTRUCTURE ONLY: restatements of the two attention kernels (plain torch, no product imports).

Three functions, from the semantics down to the arithmetic:
  * softmax_attention_fp64: what af3_attention / af3_decode_attention compute (include/af3b200.h), evaluated in fp64.
    Masks: keys >= min(kv_len[b], Tk) and keys < kv_start[b] are invisible; causal keeps key j for query i iff
    j <= i + (Tk - Tq).  GQA: query head h reads KV head h // (H / Hkv).  A row with no visible key gives 0.
    It also returns the per-element bound  B = sum_j p_j |v_j| / sum_j p_j  that scales the rounding error of P . V,
    the largest score magnitude  A = max_j sum_d |q_d k_jd| * scale  of each row, which bounds the fp32 score error, and
    W = max_j (p_j / sum p) * max_j |v_jd|, which bounds what one P rounding that falls the other way can move.
  * prefill_tile_restatement: attention_kernel<D, NWG> (attention_wgmma.cu) step by step -- 128-key tiles at absolute
    multiples of 128, log2-domain running maximum, P rounded to bf16 for P . V while the denominator sums the unrounded P.
  * decode_split_restatement: decode_attn_kernel (decode_attention.cu) -- the live 128-key chunks divided over nz splits,
    an online softmax inside each split, and the log-sum-exp merge of combine_heads.
With rounding=False the restatements drop every rounding point (fp32 scores, bf16 P, fp32 scale, bf16 output) and
reduce to softmax_attention_fp64 up to fp64 error.

Layouts: q [B, Tq, H, D] (decode: [B, H, D]); k, v [B, Hkv, Tk, D] (the cache layout; decode reads [0, ctx)).
Everything is computed per (batch, KV head) so that the fp64 score blocks stay small.

Also here: the score profiles the tests use (peak_scores, edge_probe, diagonal_probe).
"""
from __future__ import annotations

import math

import torch

TILE = 128                          # keys per tile (prefill) / per chunk (decode)
LOG2E_F32 = 1.4426950408889634      # the kernels' constant, as an fp32 literal
F64 = torch.float64


def _ints(x, B, default):
    if x is None:
        return [default] * B
    return [int(t) for t in (x.tolist() if torch.is_tensor(x) else x)]


def visible_mask(B, Tq, Tk, causal, kv_len=None, kv_start=None, device="cpu"):
    """bool [B, Tq, Tk]: True where query i may read key j (the af3_attention header's rules)."""
    lens = [min(n, Tk) for n in _ints(kv_len, B, Tk)]
    starts = _ints(kv_start, B, 0)
    j = torch.arange(Tk, device=device)
    i = torch.arange(Tq, device=device)
    m = torch.stack([(j >= s) & (j < n) for s, n in zip(starts, lens)])[:, None, :].expand(B, Tq, Tk).clone()
    if causal:
        m &= (j[None, :] <= i[:, None] + (Tk - Tq))[None]
    return m


def _f32_scale_log2(scale):
    return float(torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E_F32, dtype=torch.float32))


def _exp2_f32(x):
    """ex2.approx.ftz.f32 up to its ~2^-22 error: 2^x rounded to fp32, results below 2^-126 flushed to +0."""
    y = torch.exp2(x.to(F64))
    return torch.where(y < 2.0 ** -126, torch.zeros_like(y), y).float()


def softmax_attention_fp64(q, k, v, scale, causal=False, kv_len=None, kv_start=None):
    """-> (out, bnd, smag, wmax): out, bnd and wmax fp64 [B, Tq, H, D], smag fp64 [B, Tq, H]."""
    B, Tq, H, D = q.shape
    Hkv, Tk = k.shape[1], k.shape[2]
    G = H // Hkv
    vis = visible_mask(B, Tq, Tk, causal, kv_len, kv_start, q.device)
    out = torch.zeros((B, Tq, H, D), dtype=F64, device=q.device)
    bnd = torch.zeros_like(out)
    smag = torch.zeros((B, Tq, H), dtype=F64, device=q.device)
    wmax = torch.zeros_like(out)
    for b in range(B):
        m = vis[b][None]                                            # [1, Tq, Tk]
        for hk in range(Hkv):
            qh = q[b, :, hk * G:(hk + 1) * G].to(F64).transpose(0, 1)  # [G, Tq, D]
            kh, vh = k[b, hk].to(F64), v[b, hk].to(F64)
            s = torch.where(m, (qh @ kh.T) * scale, -math.inf)
            mx = s.amax(-1, keepdim=True)
            p = torch.where(m, torch.exp(s - torch.where(mx == -math.inf, 0.0, mx)), 0.0)
            l = p.sum(-1, keepdim=True)
            inv = torch.where(l > 0, 1.0 / l, 0.0)
            out[b, :, hk * G:(hk + 1) * G] = ((p @ vh) * inv).transpose(0, 1)
            bnd[b, :, hk * G:(hk + 1) * G] = ((p @ vh.abs()) * inv).transpose(0, 1)
            a = torch.where(m, qh.abs() @ kh.abs().T, 0.0).amax(-1) * abs(scale)
            smag[b, :, hk * G:(hk + 1) * G] = a.transpose(0, 1)
            w = (p * inv).amax(-1)[..., None] * vh.abs().amax(0)
            wmax[b, :, hk * G:(hk + 1) * G] = w.transpose(0, 1)
    return out, bnd, smag, wmax


def attention_tolerance(ref, bnd, smag, D, n_keys, extra=0.0):
    """Per-element bound on |kernel - ref| (see the docstring of tests/test_attention_kernels_gpu.py):
        2^-8 (B + |ref|) (1 + slack) + 2^-126,   slack = 2^8 eps + 2^-7,
        eps = 2 (D + 4) 2^-24 A + (n_tiles + 2) 2^-22 + 2 n_keys 2^-24 + extra.
    2^-8 B: P rounded to bf16 (the denominator sums the unrounded P); 2^-8 |ref|: the bf16 output.  eps bounds the relative
    error of each weight from the fp32 score (A = the row's largest sum |q k| scale), the fp32 exponent and ex2.approx, plus
    the fp32 accumulation of P . V and of the denominator over n_keys terms."""
    n_tiles = -(-n_keys // TILE)
    eps = 2 * (D + 4) * 2.0 ** -24 * smag[..., None] + (n_tiles + 2) * 2.0 ** -22 + 2 * n_keys * 2.0 ** -24 + extra
    slack = 2.0 ** 8 * eps + 2.0 ** -7
    return 2.0 ** -8 * (bnd + ref.abs()) * (1 + slack) + 2.0 ** -126


def prefill_tile_restatement(q, k, v, scale, causal=False, kv_len=None, kv_start=None, rounding=True):
    """attention_kernel's arithmetic -> bf16 [B, Tq, H, D] (fp64 with rounding=False).  Every tile of every row is
    visited: a tile a CTA visits but that is fully masked for a row is a no-op in the kernel (alpha = 1, p = 0), so the
    result does not depend on the row tiling."""
    B, Tq, H, D = q.shape
    Hkv, Tk = k.shape[1], k.shape[2]
    G = H // Hkv
    sl2 = _f32_scale_log2(scale) if rounding else scale * math.log2(math.e)
    vis = visible_mask(B, Tq, Tk, causal, kv_len, kv_start, q.device)
    out = torch.zeros((B, Tq, H, D), dtype=F64, device=q.device)
    for b in range(B):
        for hk in range(Hkv):
            qh = q[b, :, hk * G:(hk + 1) * G].to(F64).transpose(0, 1)
            kh, vh = k[b, hk].to(F64), v[b, hk].to(F64)
            s = qh @ kh.T
            if rounding:
                s = s.float()                                        # fp32 wgmma accumulator
            s = torch.where(vis[b][None], s, -math.inf)
            m_run = torch.full((G, Tq), -math.inf, dtype=s.dtype, device=q.device)
            l_run = torch.zeros((G, Tq), dtype=F64, device=q.device)
            o = torch.zeros((G, Tq, D), dtype=F64, device=q.device)
            for k0 in range(0, Tk, TILE):
                st = s[..., k0:k0 + TILE]
                mx = st.amax(-1)
                m_new = torch.maximum(m_run, mx * sl2)               # fp32 product when rounding
                if rounding:
                    alpha = torch.where(m_run == -math.inf, 0.0, _exp2_f32(m_run - m_new).to(F64))
                    neg_m = torch.where(m_new == -math.inf, 0.0, -m_new).to(F64)
                    x = (st.to(F64) * sl2 + neg_m[..., None]).float()   # fmaf(s, sl2, -m)
                    p = _exp2_f32(x).to(F64)
                else:
                    alpha = torch.where(m_run == -math.inf, 0.0, torch.exp2(m_run - m_new))
                    neg_m = torch.where(m_new == -math.inf, 0.0, -m_new)
                    p = torch.exp2(st * sl2 + neg_m[..., None])
                m_run = m_new
                l_run = l_run * alpha + p.sum(-1)
                pr = p.bfloat16().to(F64) if rounding else p
                o = o * alpha[..., None] + pr @ vh[k0:k0 + TILE]
            res = torch.where(l_run[..., None] > 0, o / torch.where(l_run > 0, l_run, 1.0)[..., None], 0.0)
            out[b, :, hk * G:(hk + 1) * G] = res.transpose(0, 1)
    return out.bfloat16() if rounding else out


def decode_splits(B, Hkv, Tmax, sm_count, override=None):
    """The host's split count (pick_splits): SMs / (B Hkv), or the override, clamped to [1, chunks(Tmax)]."""
    nz = override if override else sm_count // (B * Hkv)
    return max(1, min(nz, -(-Tmax // TILE)))


def decode_split_restatement(q, k, v, scale, ctx, kv_start=None, nz=1, rounding=True):
    """decode_attn_kernel's arithmetic for q [B, H, D] over cache rows [kv_start[b], ctx) -> bf16 [B, H, D]
    (fp64 with rounding=False)."""
    B, H, D = q.shape
    Hkv = k.shape[1]
    G = H // Hkv
    sl2 = _f32_scale_log2(scale) if rounding else scale * math.log2(math.e)
    starts = _ints(kv_start, B, 0)
    out = torch.zeros((B, H, D), dtype=F64, device=q.device)
    for b in range(B):
        start = starts[b]
        c_lo, c_hi = start // TILE, -(-ctx // TILE)
        n_live = max(c_hi - c_lo, 0)
        cps = -(-n_live // nz)
        n_used = -(-n_live // cps) if cps else 0
        for hk in range(Hkv):
            qh = q[b, hk * G:(hk + 1) * G].to(F64)                  # [G, D]
            parts = []
            for sp in range(n_used):
                c_beg = c_lo + sp * cps
                m_run = torch.full((G,), -math.inf, dtype=torch.float32 if rounding else F64, device=q.device)
                l_run = torch.zeros((G,), dtype=F64, device=q.device)
                acc = torch.zeros((G, D), dtype=F64, device=q.device)
                for c in range(c_beg, min(c_hi, c_beg + cps)):
                    j = torch.arange(c * TILE, (c + 1) * TILE, device=q.device)
                    kc, vc = k[b, hk, c * TILE:(c + 1) * TILE].to(F64), v[b, hk, c * TILE:(c + 1) * TILE].to(F64)
                    valid = (j >= start) & (j < ctx)
                    s = qh @ kc.T                                    # [G, 128]
                    t = (s.float() * sl2) if rounding else s * sl2   # fp32(fp32(s) * scale_log2)
                    t = torch.where(valid[None], t, -math.inf)
                    m_new = torch.maximum(m_run, t.amax(-1))
                    if rounding:
                        a = torch.where(m_run == -math.inf, 0.0, _exp2_f32(m_run - m_new).to(F64))
                        p = torch.where(t == -math.inf, 0.0, _exp2_f32(t - m_new[:, None]).to(F64))
                    else:
                        a = torch.where(m_run == -math.inf, 0.0, torch.exp2(m_run - m_new))
                        p = torch.where(t == -math.inf, 0.0, torch.exp2(t - m_new[:, None]))
                    l_run = l_run * a + p.sum(-1)
                    pr = p.bfloat16().to(F64) if rounding else p
                    vz = torch.where(valid[:, None], vc, 0.0)        # p = 0 there; keeps 0 * 1e30 out of fp64
                    acc = acc * a[:, None] + pr @ vz
                    m_run = m_new
                parts.append((acc, m_run.to(F64), l_run))
            if not parts:
                continue
            if nz == 1:
                res = acc / l_run[:, None]
            else:
                m = torch.stack([pm for _, pm, _ in parts]).amax(0)
                o = torch.zeros((G, D), dtype=F64, device=q.device)
                l = torch.zeros((G,), dtype=F64, device=q.device)
                for acc_s, m_s, l_s in parts:
                    w = torch.exp2(m_s - m)
                    if rounding:
                        w = w.float().to(F64)                        # exp2f
                    l = l + w * l_s
                    o = o + w[:, None] * acc_s
                res = o * (1.0 / l)[:, None]
            out[b, hk * G:(hk + 1) * G] = res
    return out.bfloat16() if rounding else out


# ----------------------------------------------------------------------------------------------- score profiles
def peak_scores(q, k, kind, scale, first, last, j):
    """Overwrite q (every head = e_0) and k[..., 0] so that the attention score of the key at position j is a chosen profile
    (natural-log units): 'rising' climbs by 20 per 128 keys up to the key at `last` (the running maximum moves every chunk and
    the online-softmax rescale is << 1), 'falling' is its mirror (maximum at `first`), 'two_peaks' has equal peaks at `first` and
    `last` and falls by 0.3 per key between them (partials whose maxima differ by hundreds).  'random' leaves both alone."""
    if kind == "random":
        return
    if kind == "rising":
        f = 20 / 128 * (j - last)
    elif kind == "falling":
        f = -20 / 128 * (j - first)
    else:
        f = -0.3 * torch.minimum((j - first).abs(), (j - last).abs())
    q.zero_()
    q[..., 0] = 1.0
    k[..., 0] = (f / scale).to(k.dtype)


def edge_probe(q, k, v, scale, masked, visible, hi=12.0, lo=8.0):
    """Boundary probe on random q / k / v: feature 0 of every query is 1 (in score units: q_0 = 1, k_0 = score / scale);
    the keys in `masked` (the first key each masking rule removes) get score +hi and v = +3, -1.5 (in that order), the
    keys in `visible` (the last key each rule keeps) get +lo and v = -3, +1.5.  A one-key leak pulls the output towards a
    masked key's value, a drop towards the other visible key's value or the random rest: both far beyond the tolerance.
    q [..., D], k / v [Tk, D] (one sequence's keys); positions outside [0, Tk) are skipped."""
    Tk = k.shape[0]
    q[..., 0] = 1.0
    k[:, 0] = 0.0
    for pos, sc, val in list(zip(visible, (lo, lo), (-3.0, 1.5))) + list(zip(masked, (hi, hi), (3.0, -1.5))):
        if 0 <= pos < Tk:
            k[pos, 0] = sc / scale
            v[pos] = val


DIAG_FREQS = 10


def diagonal_probe(q, k, scale, off, c=10.0):
    """Causal-diagonal probe: query i's highest score is the first key the causal rule removes (j = i + off + 1), the
    next ones its last visible key and the key after the peak.  Features 2f, 2f + 1 hold a rotation by theta_f = 2^-f rad:
        q_i = c / scale [cos theta_f (i + off + 1), sin ...],   k_j = [cos theta_f j, sin theta_f j],
        score(i, j) = c sum_f cos(theta_f (i + off + 1 - j)),
    largest at j = i + off + 1 and lower by c sum_f (1 - cos theta_f) ~ 0.62 c at its neighbours.  The slowest
    rotation (2^-9 rad) keeps every |i + off + 1 - j| < 1600 away from a second peak.  Scores stay within c * 10.
    q [Tq, H, D] (every head alike), k [Tk, Hkv, D]; the other features are zeroed."""
    Tq, Tk = q.shape[0], k.shape[0]
    th = 2.0 ** -torch.arange(DIAG_FREQS, dtype=F64)
    ai = (torch.arange(Tq, dtype=F64)[:, None] + off + 1) * th
    aj = torch.arange(Tk, dtype=F64)[:, None] * th
    qf = torch.stack([ai.cos(), ai.sin()], -1).reshape(Tq, 2 * DIAG_FREQS) * (c / scale)
    kf = torch.stack([aj.cos(), aj.sin()], -1).reshape(Tk, 2 * DIAG_FREQS)
    q.zero_()
    k.zero_()
    q[..., :2 * DIAG_FREQS] = qf[:, None, :].to(q.device, q.dtype)
    k[..., :2 * DIAG_FREQS] = kf[:, None, :].to(k.device, k.dtype)
