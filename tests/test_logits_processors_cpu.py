"""Host-side compiler of the greedy logits processors (audio_flamingo_b200/logits_process.py) against the reference's own
processor construction ([O] generation/utils.py _get_logits_processor, [O] generation/logits_process.py), without a GPU:
option resolution, validation errors, EOS filtering of bad words, begin_index, the forced-EOS step, and the compiled tables
evaluated by a plain torch restatement of the kernels' rules == LogitsProcessorList on random CPU inputs."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from audio_flamingo_b200 import logits_process as LP


def ref_chain(opts, eos, S, max_length, device="cpu"):
    """The reference's LogitsProcessorList for a greedy call with prompt length S (what generate() builds)."""
    from transformers import GenerationConfig
    from transformers.generation.utils import GenerationMixin

    gc = GenerationConfig(max_length=max_length, **{k: v for k, v in opts.items() if v is not None})
    if gc.min_new_tokens is not None:
        gc.min_length = gc.min_new_tokens + S          # _prepare_generated_length
    gc._eos_token_tensor = torch.tensor(eos, device=device) if eos is not None else None
    me = SimpleNamespace(_merge_criteria_processor_list=lambda p, extra: p)
    return GenerationMixin._get_logits_processor(me, gc, input_ids_seq_length=S, device=device)


def eval_tables(c, hist, logits):
    """Plain restatement of csrc/elementwise.cu logits_rules_kernel + logits_process_partial_kernel on the compiled tables."""
    t = c.tables.tolist()
    h = t[:LP.HDR]
    S, cur = h[LP.H_S], hist.shape[1]
    gen = cur - S
    V = logits.shape[1]
    static = torch.from_numpy(c.static_add)
    f32 = lambda bits: np.array([bits], dtype=np.int32).view(np.float32)[0]  # noqa: E731
    out = torch.empty_like(logits)
    for b in range(logits.shape[0]):
        x, hs = logits[b], hist[b].tolist()
        if h[LP.H_FORCED] >= 0 and cur == h[LP.H_FORCED]:
            r = torch.full((V,), -float("inf"))
            for i in range(h[LP.H_NFORCED]):
                tok, fl = t[h[LP.H_OFORCED] + 2 * i: h[LP.H_OFORCED] + 2 * i + 2]
                sup = (fl & 1) or ((fl & 2) and cur == h[LP.H_BEGIN])
                r[tok] = -float("inf") if sup else 0.0
            out[b] = r
            continue
        r = x + static if h[LP.H_STATIC] else x.clone()
        masked, adds = set(), {}
        n = h[LP.H_NGRAM]
        if n > 0 and cur + 1 >= n:
            pre = hs[cur - n + 1:]
            for j in range(cur - n + 1):
                if hs[j:j + n - 1] == pre and 0 <= hs[j + n - 1] < V:
                    masked.add(hs[j + n - 1])
        for i in range(h[LP.H_NBAD]):
            off, L = t[h[LP.H_OBAD] + 2 * i: h[LP.H_OBAD] + 2 * i + 2]
            seq = t[off:off + L]
            if L <= cur and hs[cur - L + 1:] == seq[:-1]:
                masked.add(seq[-1])
        for i in range(h[LP.H_NGRP]):
            tok, sb, mo, mc = t[h[LP.H_OGRP] + 4 * i: h[LP.H_OGRP] + 4 * i + 4]
            total, any_ = np.float32(0.0) + f32(sb), False
            for m in range(mc):
                off, L, bb = t[mo + 3 * m: mo + 3 * m + 3]
                seq = t[off:off + L]
                if L <= cur and hs[cur - L + 1:] == seq[:-1]:
                    total, any_ = np.float32(total + f32(bb)), True
            if any_:
                adds[tok] = total
        if cur < h[LP.H_MINLEN] or gen < h[LP.H_MINNEW]:
            masked.update(t[h[LP.H_OEOS]: h[LP.H_OEOS] + h[LP.H_NEOS]])
        if cur == h[LP.H_BEGIN]:
            masked.update(t[h[LP.H_OBEGIN]: h[LP.H_OBEGIN] + h[LP.H_NBEGIN]])
        for tok, tot in adds.items():
            r[tok] = -float("inf") if static[tok] == -float("inf") else x[tok] + torch.tensor(tot)
        if masked:
            r[sorted(masked)] = -float("inf")
        out[b] = r
    return out


def _opts(**kw):
    return {**{k: None for k in LP.OPTIONS + ("forced_bos_token_id",)}, **kw}


def test_defaults_compile_to_no_processors():
    assert LP.compile_processors(_opts(), [2], 10, 20, 64, 256) is None
    assert LP.compile_processors(_opts(no_repeat_ngram_size=0, min_length=0), [2], 10, 20, 64, 256) is None
    # min-length options need EOS ids, as in the reference
    assert LP.compile_processors(_opts(min_length=30, min_new_tokens=5), None, 10, 20, 64, 256) is None
    assert len(ref_chain(_opts(min_length=30, min_new_tokens=5), None, 10, 20)) == 0


def test_resolve_options_argument_then_config():
    gc = {"no_repeat_ngram_size": 3, "suppress_tokens": [1, 2]}
    o = LP.resolve_options({"no_repeat_ngram_size": 2, "bad_words_ids": None}, gc.get)
    assert o["no_repeat_ngram_size"] == 2 and o["suppress_tokens"] == [1, 2] and o["bad_words_ids"] is None


def test_sequence_bias_formats_compile_alike():
    d = {(5,): 1.5, (3, 7): -2.0, (4, 7): 0.25, (7,): 0.5}
    lst = [[[5], 1.5], [[3, 7], -2.0], [[4, 7], 0.25], [[7], 0.5]]
    a = LP.compile_processors(_opts(sequence_bias=d), None, 6, 20, 16, 64)
    b = LP.compile_processors(_opts(sequence_bias=lst), None, 6, 20, 16, 64)
    assert np.array_equal(a.tables, b.tables) and np.array_equal(a.static_add, b.static_add)
    assert a.static_add[5] == np.float32(1.5) and a.static_add[7] == np.float32(0.5)
    assert a.tables[LP.H_NGRP] == 1   # both 2-token sequences end in 7: one group, members in dict order


def test_bad_words_eos_filter_begin_index_and_forced_step():
    c = LP.compile_processors(_opts(bad_words_ids=[[2], [9], [4, 2]]), [2], 6, 20, 16, 64)
    assert c.static_add[2] == 0 and c.static_add[9] == -np.inf and c.tables[LP.H_NBAD] == 1
    c = LP.compile_processors(_opts(bad_words_ids=[[2]]), [2], 6, 20, 16, 64)    # every entry filtered: a processor without rules
    assert not c.static_add.any() and c.tables[LP.H_STATIC] == 0 and c.tables[LP.H_NBAD] == 0
    c = LP.compile_processors(_opts(begin_suppress_tokens=[3], forced_eos_token_id=[2, 5, 2], suppress_tokens=[5]), [2], 6, 20, 16, 64)
    assert c.tables[LP.H_BEGIN] == 6 and c.tables[LP.H_FORCED] == 19 and c.tables[LP.H_NFORCED] == 2
    # S == 1 with a forced BOS id moves begin_index by one ([O] utils.py:1180-1185)
    c = LP.compile_processors(_opts(begin_suppress_tokens=[3], forced_bos_token_id=1), None, 1, 20, 16, 64)
    assert c.tables[LP.H_BEGIN] == 2


@pytest.mark.parametrize("bad", [
    dict(sequence_bias={}), dict(sequence_bias=[]), dict(sequence_bias={(1, -2): 1.0}), dict(sequence_bias={(1,): 1}),
    dict(sequence_bias={5: 1.0}), dict(sequence_bias=[[[0], 1.0]]), dict(sequence_bias={(99,): 1.0}),
    dict(bad_words_ids=[]), dict(bad_words_ids=[1, 2]), dict(bad_words_ids=[[1, -3]]),
    dict(bad_words_ids=[[3, 99]]), dict(no_repeat_ngram_size=2.5), dict(min_length=2.5), dict(min_new_tokens=1.5),
    dict(forced_eos_token_id=-1),
])
def test_validation_errors_match_the_reference(bad):
    """Same malformed input -> ValueError in the reference's construction / first call and in compile_processors."""
    V, S, eos = 16, 4, [2]
    ids, scores = torch.zeros((1, S), dtype=torch.long), torch.zeros((1, V))
    with pytest.raises(ValueError):
        ref_chain(_opts(**bad), eos, S, 20)(ids, scores)
    with pytest.raises(ValueError):
        LP.compile_processors(_opts(**bad), eos, S, 20, V, 64)


def _random_case(rs, V):
    eos = [int(x) for x in rs.choice(V, size=rs.randint(1, 3), replace=False)]
    toks = lambda n: [int(x) for x in rs.randint(0, 8, size=n)]  # noqa: E731  (a small alphabet: repeats and matches happen)
    return eos, dict(
        sequence_bias={(int(rs.randint(V)),): float(rs.randn()), tuple(toks(2)): float(rs.randn()), tuple(toks(3)): float(rs.randn()),
                       tuple(toks(1) + [3]): 2.0, tuple(toks(2) + [3]): -1.0},
        no_repeat_ngram_size=int(rs.randint(1, 4)),
        bad_words_ids=[toks(1), toks(2), toks(3), [eos[0]]],
        min_length=int(rs.randint(0, 12)),
        min_new_tokens=int(rs.randint(0, 4)) if rs.rand() < 0.5 else None,
        forced_eos_token_id=eos if rs.rand() < 0.5 else None,
        suppress_tokens=[int(x) for x in rs.choice(V, size=3, replace=False)],
        begin_suppress_tokens=[int(x) for x in rs.choice(V, size=2, replace=False)],
    )


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("only", [None, *LP.OPTIONS])
def test_tables_restated_equal_reference_chain(seed, only):
    rs = np.random.RandomState(seed)
    V, B, S, new = 24, 3, 5, 8
    eos, opts = _random_case(rs, V)
    if only is not None:
        opts = {only: opts[only]}
    opts = _opts(**opts)
    c = LP.compile_processors(opts, eos, S, S + new, V, 64)
    chain = ref_chain(opts, eos, S, S + new)
    hist = torch.from_numpy(rs.randint(0, 8, size=(B, S + new)).astype(np.int64))
    for i in range(new):
        cur = hist[:, :S + i]
        logits = torch.from_numpy(rs.randn(B, V).astype(np.float32)).to(torch.bfloat16).float()
        ref = chain(cur, logits)
        got = eval_tables(c, cur, logits) if c is not None else logits
        assert torch.equal(got, ref), (only, i)
