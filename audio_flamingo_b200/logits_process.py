"""Host side of the greedy logits processors (include/af3b200.h af3_logits_process_argmax).

`resolve_options` collects the processor options of `generate()` (argument, else generation config), and
`compile_processors` validates them where the reference does ([O] generation/logits_process.py constructors and
SequenceBiasLogitsProcessor._prepare_bias_variables; same inputs -> the same ValueError, raised before anything is enqueued) and
compiles them into the int32 tables and the fp32 static vector the kernels read.  The chain is the one
[O] generation/utils.py:1037-1192 _get_logits_processor builds for greedy decoding:
    sequence_bias -> no_repeat_ngram_size -> bad_words_ids -> min_length -> min_new_tokens -> forced_eos_token_id
    -> suppress_tokens -> begin_suppress_tokens
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

OPTIONS = ("sequence_bias", "no_repeat_ngram_size", "bad_words_ids", "min_length", "min_new_tokens", "forced_eos_token_id",
           "suppress_tokens", "begin_suppress_tokens")

# table header (csrc/elementwise.cu LP_*)
(H_S, H_NGRAM, H_MINLEN, H_MINNEW, H_BEGIN, H_FORCED, H_STATIC, H_NEOS, H_OEOS, H_NBEGIN, H_OBEGIN, H_NFORCED, H_OFORCED, H_NBAD, H_OBAD,
 H_NGRP, H_OGRP) = range(17)
HDR = 32
FORCED_SUPPRESSED, FORCED_BEGIN_SUPPRESSED = 1, 2


@dataclass
class Compiled:
    tables: np.ndarray        # int32 [n]: header + records (layout above and in csrc/elementwise.cu)
    static_add: np.ndarray    # fp32 [V]: single-token bias, -inf for single-token bad words and suppress_tokens
    cap: int                  # rule-list entries per row the kernels may need


def _is_int(x):
    return isinstance(x, (int, np.integer)) and not isinstance(x, bool)


def resolve_options(kwargs, default):
    """Processor options: the argument when given (not None), else `default(name)` (the generation config)."""
    return {k: (kwargs[k] if kwargs.get(k) is not None else default(k)) for k in OPTIONS + ("forced_bos_token_id",)}


def _bias_dict(sequence_bias):
    """SequenceBiasLogitsProcessor._validate_arguments + _convert_list_arguments_into_dict."""
    sb = sequence_bias
    if not isinstance(sb, dict) and not isinstance(sb, list) or len(sb) == 0:
        raise ValueError(f"`sequence_bias` has to be a non-empty dictionary, or non-empty list of lists but is {sb}.")
    if isinstance(sb, dict):
        if any(not isinstance(k, tuple) for k in sb):
            raise ValueError(f"`sequence_bias` has to be a dict with tuples as keys, but is {sb}.")
        if any(any((not _is_int(t) or t < 0) for t in k) or len(k) == 0 for k in sb):
            raise ValueError(f"Each key in `sequence_bias` has to be a non-empty tuple of positive integers, but is {sb}.")
        if any(not isinstance(v, float) for v in sb.values()):
            raise ValueError(f"`sequence_bias` has to be a dict with floats as values, but is {sb}.")
        return dict(sb)

    def pair_ok(s):
        return isinstance(s[0], list) and all(_is_int(t) and t > 0 for t in s[0]) and isinstance(s[1], float)

    if any((not pair_ok(s)) or len(s) == 0 for s in sb):
        raise ValueError(f"Each element in `sequence_bias` has to be a non-empty list of lists of positive integers and float, but is {sb}.")
    return {tuple(s[0]): s[1] for s in sb}


def _bad_words_dict(bad_words_ids, eos):
    """NoBadWordsLogitsProcessor.__init__: validation, then EOS single-token entries dropped (what remains may be empty)."""
    bw = bad_words_ids
    if not isinstance(bw, list) or len(bw) == 0:
        raise ValueError(f"`bad_words_ids` has to be a non-empty list, but is {bw}.")
    if any(not isinstance(w, list) for w in bw):
        raise ValueError(f"`bad_words_ids` has to be a list of lists, but is {bw}.")
    if any(any((not _is_int(t) or t < 0) for t in w) for w in bw):
        raise ValueError(f"Each list in `bad_words_ids` has to be a list of positive integers, but is {bw}.")
    if eos is not None:
        bw = [w for w in bw if all(w != [i] for i in eos)]
    if any(len(w) == 0 for w in bw):
        raise ValueError(f"Each list in `bad_words_ids` has to be non-empty, but is {bw}.")
    return {tuple(w): float("-inf") for w in bw}


def _check_vocab(d, V):
    """SequenceBiasLogitsProcessor._prepare_bias_variables (first call): biased ids must lie in the vocabulary."""
    bad = [t for k in d for t in k if t >= V]
    if bad:
        raise ValueError(f"The model vocabulary size is {V}, but the following tokens were being biased: {bad}")


def _nonneg_int(name, v, positive_msg=False):
    if not _is_int(v) or v < 0:
        raise ValueError(f"`{name}` has to be a {'positive' if positive_msg else 'non-negative'} integer, but is {v}")


def compile_processors(opts, eos, S, max_length, V, Tmax):
    """Validates `opts` (from resolve_options) and compiles them for a call with prompt length S, max_length = S +
    max_new_tokens, vocabulary V and history capacity Tmax.  eos: list of EOS ids or None.  Returns None when the reference
    would build no processor (every option at its default): the caller then runs the plain argmax."""
    sb = opts.get("sequence_bias")
    ngram = opts.get("no_repeat_ngram_size")
    bw = opts.get("bad_words_ids")
    min_new = opts.get("min_new_tokens")
    min_len = opts.get("min_length")
    if min_new is not None:   # _prepare_generated_length: min_new_tokens takes precedence and is counted from the prompt
        min_len = min_new + S
    forced = opts.get("forced_eos_token_id")
    sup = opts.get("suppress_tokens")
    bsup = opts.get("begin_suppress_tokens")
    # construction, in _get_logits_processor's order
    bias = _bias_dict(sb) if sb is not None else None
    if ngram is not None and ngram > 0:
        if not _is_int(ngram):
            raise ValueError(f"`ngram_size` has to be a strictly positive integer, but is {ngram}")
    else:
        ngram = 0
    bad = _bad_words_dict(bw, eos) if bw is not None else None
    min_len_on = min_len is not None and eos is not None and min_len > 0
    if min_len_on:
        _nonneg_int("min_length", min_len)
    min_new_on = min_new is not None and eos is not None and min_new > 0
    if min_new_on:
        _nonneg_int("min_new_tokens", min_new, positive_msg=True)
    forced_ids = None
    if forced is not None:
        forced_ids = [forced] if _is_int(forced) else list(forced)
        if any(not _is_int(f) for f in forced_ids) or any(f < 0 for f in forced_ids):
            raise ValueError(f"`eos_token_id` has to be a list of positive integers, but is {forced}")
        if any(f >= V for f in forced_ids):
            raise ValueError(f"`forced_eos_token_id` {forced} lies outside the vocabulary of size {V}")
    sup_ids = [int(t) for t in sup] if sup is not None else None
    bsup_ids = [int(t) for t in bsup] if bsup is not None else None
    if bias is None and not ngram and bad is None and not min_len_on and not min_new_on and forced_ids is None and sup_ids is None \
            and bsup_ids is None:
        return None
    if bias is not None:
        _check_vocab(bias, V)
    if bad is not None:
        _check_vocab(bad, V)

    static = np.zeros((V,), dtype=np.float32)
    has_static = False
    recs = []          # (group token, single bias, [(seq, bias)]) for sequence_bias; [seq] for bad words
    if bias is not None:
        single = {k[0]: np.float32(v) for k, v in bias.items() if len(k) == 1}
        for t, v in single.items():
            static[t] = np.float32(0.0) + v
            has_static = True
        groups = {}
        for k, v in bias.items():
            if len(k) > 1:
                groups.setdefault(k[-1], []).append((k, np.float32(v)))
        recs = [(t, single.get(t, np.float32(0.0)), mem) for t, mem in groups.items()]
    bad_multi = []
    if bad is not None:
        for k in bad:
            if len(k) == 1:
                static[k[0]] = -np.inf
                has_static = True
            else:
                bad_multi.append(k)
    if sup_ids:
        ids = np.array([t for t in sup_ids if 0 <= t < V], dtype=np.int64)
        static[ids] = -np.inf
        has_static = has_static or len(ids) > 0
    in_vocab = lambda ids: sorted({t for t in ids if 0 <= t < V})  # noqa: E731  (torch.isin semantics: others never match)
    eos_mask = in_vocab(eos) if (min_len_on or min_new_on) else []
    begin = in_vocab(bsup_ids) if bsup_ids is not None else []
    # begin_index of SuppressTokensAtBeginLogitsProcessor ([O] generation/utils.py:1180-1185)
    begin_index = (S if (S > 1 or opts.get("forced_bos_token_id") is None) else S + 1) if bsup_ids is not None else -1
    forced_recs = []
    if forced_ids is not None:
        sup_set, bsup_set = set(sup_ids or ()), set(bsup_ids or ())
        for f in dict.fromkeys(forced_ids):
            forced_recs.append((f, (FORCED_SUPPRESSED if f in sup_set else 0) | (FORCED_BEGIN_SUPPRESSED if f in bsup_set else 0)))

    body = []

    def region(vals):
        off = HDR + len(body)
        body.extend(vals)
        return off

    hdr = [0] * HDR
    hdr[H_S], hdr[H_NGRAM] = S, ngram
    hdr[H_MINLEN] = min_len if min_len_on else 0
    hdr[H_MINNEW] = min_new if min_new_on else 0
    hdr[H_BEGIN] = begin_index
    hdr[H_FORCED] = max_length - 1 if forced_ids is not None else -1
    hdr[H_STATIC] = int(has_static)
    hdr[H_NEOS], hdr[H_OEOS] = len(eos_mask), region(eos_mask)
    hdr[H_NBEGIN], hdr[H_OBEGIN] = len(begin), region(begin)
    hdr[H_NFORCED], hdr[H_OFORCED] = len(forced_recs), region([x for r in forced_recs for x in r])
    # variable-length parts: sequences first, then the fixed-size records that point at them
    seq_off = {}

    def seq(k):
        if k not in seq_off:
            seq_off[k] = region(list(k))
        return seq_off[k]

    bad_flat = [x for k in bad_multi for x in (seq(k), len(k))]
    mem_offs = []
    for _, _, mem in recs:
        flat = [x for k, v in mem for x in (seq(k), len(k), int(np.float32(v).view(np.int32)))]
        mem_offs.append(region(flat))
    hdr[H_NBAD], hdr[H_OBAD] = len(bad_multi), region(bad_flat)
    grp_flat = [x for (t, s, mem), mo in zip(recs, mem_offs) for x in (t, int(np.float32(s).view(np.int32)), mo, len(mem))]
    hdr[H_NGRP], hdr[H_OGRP] = len(recs), region(grp_flat)
    tables = np.array(hdr + body, dtype=np.int64)
    if tables.max(initial=0) > np.iinfo(np.int32).max:
        raise ValueError("logits processor tables exceed int32 range")
    cap = (Tmax if ngram else 0) + len(bad_multi) + len(recs) + len(eos_mask) + len(begin) + len(forced_recs)
    return Compiled(tables=tables.astype(np.int32), static_add=static, cap=max(cap, 1))


def bucket(n, lo=64):
    """Capacities are rounded up to a power of two, so that calls with slightly different tables reuse one decode graph."""
    b = lo
    while b < n:
        b *= 2
    return b
