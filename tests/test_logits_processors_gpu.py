"""Greedy logits processors on the device (include/af3b200.h af3_logits_process_argmax) against the reference's own
LogitsProcessorList ([O] generation/logits_process.py, built by [O] generation/utils.py _get_logits_processor) on the same GPU:
  * kernel level: every option alone and all together, B in {1, 3, 32, 65}, V in {152064, 2048, 2051}, histories up to 15 360
    tokens with planted repeats; processed rows equal under torch.equal, ids == torch.argmax of the reference rows; repeated
    launches, PDL on / off and a CUDA-graph replay bit-identical to the eager launch
  * end to end on the tiny preset: scores[i] == the reference chain applied to our logits[i] and our sequences[:, :S+i], every
    appended id is that row's argmax after the pad rule; equal to HF generate() with the same options where the free runs
    coincide; with / without the CUDA graph, chunked prefill, B > 64
  * defaults launch no processor kernel; generation_config == arguments; on -> off -> on == a fresh instance
  * malformed options raise ValueError before any launch; still-unimplemented options raise AF3Error"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
OPTS = ("sequence_bias", "no_repeat_ngram_size", "bad_words_ids", "min_length", "min_new_tokens", "forced_eos_token_id",
        "suppress_tokens", "begin_suppress_tokens")


def ref_chain(opts, eos, S, max_length, device="cuda"):
    """The reference's LogitsProcessorList for a greedy call with prompt length S."""
    from transformers import GenerationConfig
    from transformers.generation.utils import GenerationMixin

    gc = GenerationConfig(max_length=max_length, **{k: v for k, v in opts.items() if v is not None})
    if gc.min_new_tokens is not None:
        gc.min_length = gc.min_new_tokens + S
    gc._eos_token_tensor = torch.tensor(eos, device=device) if eos is not None else None
    me = SimpleNamespace(_merge_criteria_processor_list=lambda p, extra: p)
    return GenerationMixin._get_logits_processor(me, gc, input_ids_seq_length=S, device=device)


class Runner:
    """Device tables + buffers of one processed selection, as generate() lays them out (history = prompt + generated)."""

    def __init__(self, opts, eos, S, max_length, V, B, Tmax, scores=True):
        from audio_flamingo_b200 import logits_process as LP

        full = {k: opts.get(k) for k in OPTS}
        full["forced_bos_token_id"] = None
        self.c = LP.compile_processors(full, eos, S, max_length, V, Tmax)
        self.S, self.Tmax = S, Tmax
        self.tables = torch.from_numpy(self.c.tables).cuda()
        self.static = torch.from_numpy(self.c.static_add).cuda()
        self.prompt = torch.zeros((B, Tmax), dtype=torch.int64, device="cuda")
        self.gen = torch.zeros((B, Tmax), dtype=torch.int64, device="cuda")
        self.gen_idx = torch.zeros((1,), dtype=torch.int32, device="cuda")
        self.scores = torch.empty((B, V), device="cuda") if scores else None
        self.out = torch.empty((B,), dtype=torch.int64, device="cuda")

    def set_history(self, hist):
        n = hist.shape[1] - self.S
        self.prompt[:, :self.S] = hist[:, :self.S]
        self.gen[:, :n] = hist[:, self.S:]
        self.gen_idx.fill_(n)

    def __call__(self, logits):
        from audio_flamingo_b200 import ops

        return ops.logits_process_argmax(logits, self.prompt, self.gen, self.gen_idx, self.tables, self.static, self.c.cap,
                                         out=self.out, scores=self.scores)


def _planted(rs, B, n, alphabet):
    """Histories from a small alphabet (n-gram repeats everywhere) with a planted repeated phrase."""
    h = rs.randint(0, alphabet, size=(B, n)).astype(np.int64)
    if n > 12:
        h[:, n - 4:] = h[:, 3:7]
    return torch.from_numpy(h).cuda()


def _logits(rs, B, V, ties=True):
    x = torch.from_numpy(rs.randn(B, V).astype(np.float32)).to(bf16).float().cuda()
    if ties:   # equal maxima in different argmax slices: the first index must win
        per = ((V + 31) // 32 + 3) & ~3
        m = x.max() + 1
        x[:, min(V - 1, per + 5)] = m
        x[:, min(V - 1, 3 * per + 1)] = m
    return x.contiguous()


def _case(rs, V, eos, S):
    a = 16   # history alphabet: the option tokens below match it
    toks = lambda n: [int(x) for x in rs.randint(0, a, size=n)]  # noqa: E731
    return dict(
        sequence_bias={(int(rs.randint(V)),): 1.25, tuple(toks(2)): 3.5, tuple(toks(3)): -0.75, (1, 2, 9): 2.0, (3, 9): 0.5,
                       (9,): -1.5, tuple(toks(40)): 1.0},
        no_repeat_ngram_size=3,
        bad_words_ids=[toks(1), toks(2), toks(3), [eos[0]], [5, 6, 7, 8]],
        min_length=S + 3,
        min_new_tokens=2,
        forced_eos_token_id=eos,
        suppress_tokens=[int(x) for x in rs.choice(V, size=min(1000, V // 2), replace=False)],
        begin_suppress_tokens=toks(3),
    )


def _check(run, chain, hist, logits):
    run.set_history(hist)
    ids = run(logits).clone()
    ref = chain(hist, logits.clone())
    assert torch.equal(run.scores, ref)
    assert torch.equal(ids, torch.argmax(ref, -1))
    return ids


@pytest.mark.parametrize("B,V", [(1, 152064), (3, 2048), (32, 152064), (65, 2051), (65, 2048)])
@pytest.mark.parametrize("only", [None, *OPTS])
def test_kernel_equals_reference_chain(B, V, only):
    rs = np.random.RandomState(B * 7 + V % 97)
    eos = [2, 11]
    S, new = 9, 6
    opts = _case(rs, V, eos, S)
    if only is not None:
        opts = {only: opts[only]}
    Tmax = 256
    run = Runner(opts, eos, S, S + new, V, B, Tmax)
    chain = ref_chain(opts, eos, S, S + new)
    hist = _planted(rs, B, S + new, 16)
    for cur in range(S, S + new):   # every step incl. the first (cur == S: begin index) and the forced-EOS step
        _check(run, chain, hist[:, :cur].contiguous(), _logits(rs, B, V))


@pytest.mark.parametrize("n", [1, 2, 4, 40])
def test_ngram_edges_and_long_history(n):
    """n = 1 (every earlier token banned), n longer than the history, histories of 1 .. 15 360 tokens."""
    rs = np.random.RandomState(n)
    B, V = 3, 2048
    for S, cur in [(1, 1), (1, 2), (30, 35), (15000, 15360)]:
        opts = {"no_repeat_ngram_size": n, "sequence_bias": {tuple(int(x) for x in rs.randint(0, 16, size=50)): 1.0, (3, 4): 2.0}}
        run = Runner(opts, None, S, 15361, V, B, 15360)
        chain = ref_chain(opts, None, S, 15361)
        _check(run, chain, _planted(rs, B, cur, 16 if cur < 100 else 400), _logits(rs, B, V))


def test_forced_eos_suppressed_gives_all_inf_row_and_id_zero():
    V, B, S = 2048, 3, 5
    rs = np.random.RandomState(1)
    for opts in ({"forced_eos_token_id": [7, 9, 700]},
                 {"forced_eos_token_id": [7, 9], "suppress_tokens": [7, 9]},
                 {"forced_eos_token_id": [7, 9], "suppress_tokens": [9], "begin_suppress_tokens": [7]}):
        for new in (1, 3):
            run = Runner(opts, [7], S, S + new, V, B, 64)
            chain = ref_chain(opts, [7], S, S + new)
            ids = _check(run, chain, _planted(rs, B, S + new - 1, 16), _logits(rs, B, V))
            if "suppress_tokens" in opts and len(opts["suppress_tokens"]) == 2:
                assert bool((run.scores == -float("inf")).all()) and bool((ids == 0).all())


def test_repeat_pdl_and_graph_bit_identical():
    from audio_flamingo_b200 import _lib

    rs = np.random.RandomState(5)
    B, V, S = 32, 152064, 780
    eos = [2]
    opts = _case(rs, V, eos, S)
    run = Runner(opts, eos, S, S + 200, V, B, 1024)
    hist = _planted(rs, B, S + 128, 16)
    logits = _logits(rs, B, V)
    run.set_history(hist)
    ids0, sc0 = run(logits).clone(), run.scores.clone()
    for pdl in (0, 1, 0):
        _lib.load().af3_set_pdl(pdl)
        try:
            for _ in range(3):
                assert torch.equal(run(logits), ids0) and torch.equal(run.scores, sc0)
        finally:
            _lib.load().af3_set_pdl(0)
    g = torch.cuda.CUDAGraph()
    run.scores.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(logits)
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(g):
        run(logits)
    run.scores.zero_()
    run.out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(run.out, ids0) and torch.equal(run.scores, sc0)


# ------------------------------------------------------------------------------------------------ end to end (tiny preset)
@pytest.fixture(scope="module")
def O():
    from oracle import af3_oracle

    return af3_oracle


@pytest.fixture(scope="module")
def tiny(O):
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model("tiny", seed=3, sharpen=8.0)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda")
    ref16 = O.hf_restore_fp32_rotary(O.hf_model("tiny", seed=3, sharpen=8.0).to("cuda", bf16))
    return ref32.config, ours, ref16


def _audio_inputs(O, cfg, secs, seed=1):
    waves = O.synth_waveforms(len(secs), secs, seed=seed)
    feats, fmask = O.hf_features(waves)
    toks = [O.post_pool_len(int(n)) for n in fmask.sum(-1)]
    ids, am = O.synth_prompt(toks, cfg.text_config.vocab_size, cfg.audio_token_id, seed=seed + 1)
    return feats, fmask, ids, am


def _kw(feats, fmask, ids, am, ref=False):
    f = feats.cuda().to(bf16) if ref else feats.cuda()
    return dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=f, input_features_mask=fmask.cuda())


def _option_sets(free, S, V):
    """Options drawn from the rows' own free run, so that they bite."""
    g = free[:, S:]
    t0, t1, t2 = int(g[0, 0]), int(g[0, 1]), int(g[0, 2])
    eos = list(dict.fromkeys(int(g[b, min(3, g.shape[1] - 1)]) for b in range(g.shape[0])))[:4]   # at most 8 EOS ids
    sets = {
        "ngram2": dict(no_repeat_ngram_size=2),
        "ngram3": dict(no_repeat_ngram_size=3),
        "bad_words": dict(bad_words_ids=[[t0], [t1, t2], [int(g[-1, 0])]]),
        "min_new": dict(min_new_tokens=6, eos_token_id=eos),
        "suppress": dict(suppress_tokens=[t1, t2], begin_suppress_tokens=[t0]),
        "bias": dict(sequence_bias={(t0,): -20.0, (t0, t1): -30.0, (t1, 7): 50.0}),
        "forced_eos": dict(forced_eos_token_id=[5, 6]),
    }
    allk = {}
    for v in sets.values():
        allk.update(v)
    allk["eos_token_id"] = eos
    sets["all"] = allk
    return sets


def _teacher_forced(out, opts, S, new, pad=0):
    """scores[i] == reference chain (our sequences[:, :S+i], our logits[i]); appended id == argmax, or pad after EOS."""
    eos = opts.get("eos_token_id")
    eos = [eos] if isinstance(eos, int) else eos
    chain = ref_chain({k: v for k, v in opts.items() if k in OPTS}, eos, S, S + new)
    seq = out.sequences
    assert len(out.scores) == len(out.logits) == seq.shape[1] - S
    done = torch.zeros(seq.shape[0], dtype=torch.bool, device=seq.device)
    for i, (sc, lg) in enumerate(zip(out.scores, out.logits)):
        ref = chain(seq[:, :S + i], lg.clone())
        assert torch.equal(sc, ref), f"step {i}"
        want = torch.where(done, torch.full_like(seq[:, 0], pad), torch.argmax(ref, -1))
        assert torch.equal(seq[:, S + i], want), f"step {i}"
        if eos is not None:
            done |= torch.isin(seq[:, S + i], torch.tensor(eos, device=seq.device))


def test_generate_teacher_forced_and_against_hf(O, tiny):
    cfg, ours, ref16 = tiny
    V = cfg.text_config.vocab_size
    feats, fmask, ids, am = _audio_inputs(O, cfg, [10.0, 4.3, 30.0], seed=5)
    S, new = ids.shape[1], 16
    free = ours.generate(**_kw(feats, fmask, ids, am), max_new_tokens=new).cpu()
    with torch.no_grad():
        free_ref = ref16.generate(**_kw(feats, fmask, ids, am, ref=True), max_new_tokens=new, do_sample=False).cpu()
    for name, opts in _option_sets(free, S, V).items():
        outs = []
        for graph, chunk in ((True, None), (False, None), (True, 100)):
            o = ours.generate(**_kw(feats, fmask, ids, am), max_new_tokens=new, pad_token_id=0, use_cuda_graph=graph,
                              prefill_chunk_size=chunk, return_dict_in_generate=True, output_scores=True, output_logits=True, **opts)
            assert o.past_key_values is None
            _teacher_forced(o, opts, S, new)
            outs.append(o.sequences.cpu())
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), name
        assert not torch.equal(outs[0], free), f"{name}: options changed nothing"
        plain = ours.generate(**_kw(feats, fmask, ids, am), max_new_tokens=new, pad_token_id=0, **opts)
        assert torch.equal(plain.cpu(), outs[0])
        if torch.equal(free, free_ref):
            with torch.no_grad():
                h = ref16.generate(**_kw(feats, fmask, ids, am, ref=True), max_new_tokens=new, do_sample=False, pad_token_id=0, **opts).cpu()
            print(name, "identical to HF generate:", torch.equal(h, outs[0]))
            # the free runs coincide: a row may leave the reference only through a near-tie of its processed scores
            for b in range(h.shape[0]):
                n = min(h.shape[1], outs[0].shape[1])
                diff = (h[b, S:n] != outs[0][b, S:n]).nonzero()
                if len(diff):
                    t = int(diff[0])
                    top2 = o.scores[t][b].float().topk(2).values
                    assert (top2[0] - top2[1]).item() < 0.05 * o.logits[t][b].std().item(), (name, b, t)


def test_generate_more_than_64_sequences(O, tiny):
    cfg, ours, _ = tiny
    V = cfg.text_config.vocab_size
    B, new = 70, 8
    rs = np.random.RandomState(B)
    lens = rs.randint(6, 30, size=B)
    S = int(lens.max())
    ids = torch.zeros((B, S), dtype=torch.int64)
    am = torch.zeros((B, S), dtype=torch.int64)
    for b, n in enumerate(lens):
        ids[b, S - n:] = torch.from_numpy(rs.randint(1, V - 2, size=n))
        am[b, S - n:] = 1
    free = ours.generate(input_ids=ids.cuda(), attention_mask=am.cuda(), max_new_tokens=new).cpu()
    for opts in (dict(no_repeat_ngram_size=1), _option_sets(free, S, V)["all"]):
        for graph in (True, False):
            o = ours.generate(input_ids=ids.cuda(), attention_mask=am.cuda(), max_new_tokens=new, pad_token_id=0, use_cuda_graph=graph,
                              return_dict_in_generate=True, output_scores=True, output_logits=True, **opts)
            _teacher_forced(o, opts, S, new)
        assert not torch.equal(o.sequences.cpu()[:, :free.shape[1]], free)


def _kernels(fn):
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


def test_defaults_config_and_switching(O, tiny):
    from transformers import GenerationConfig

    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    cfg, ours, _ = tiny
    feats, fmask, ids, am = _audio_inputs(O, cfg, [6.0, 3.0], seed=9)
    kw = _kw(feats, fmask, ids, am)
    names = _kernels(lambda: ours.generate(**kw, max_new_tokens=6))
    assert names and not any("logits_rules" in n or "logits_process" in n for n in names)
    names = _kernels(lambda: ours.generate(**kw, max_new_tokens=6, no_repeat_ngram_size=2))
    assert any("logits_rules" in n for n in names) and any("logits_process_partial" in n for n in names)
    # options through generation_config == the same options as arguments
    opts = dict(no_repeat_ngram_size=2, suppress_tokens=[1, 2, 3], min_new_tokens=3, eos_token_id=[4, 5])
    a = ours.generate(**kw, max_new_tokens=10, **opts)
    b = ours.generate(**kw, generation_config=GenerationConfig(max_new_tokens=10, pad_token_id=0, **opts))
    assert torch.equal(a, b)
    # on -> off -> on at one shape == a fresh instance
    off = ours.generate(**kw, max_new_tokens=10)
    on2 = ours.generate(**kw, max_new_tokens=10, **opts)
    fresh = AudioFlamingo3ForConditionalGeneration.from_reference(O.hf_model("tiny", seed=3, sharpen=8.0), device="cuda")
    assert torch.equal(on2, a) and torch.equal(on2, fresh.generate(**kw, max_new_tokens=10, **opts))
    assert torch.equal(off, fresh.generate(**kw, max_new_tokens=10))
    # scores without processors are the raw logits; output_logits == return_logits
    o = ours.generate(**kw, max_new_tokens=5, return_dict_in_generate=True, output_scores=True, output_logits=True)
    _, lg = ours.generate(**kw, max_new_tokens=5, return_logits=True)
    assert torch.equal(torch.stack(o.scores, 1), lg) and torch.equal(torch.stack(o.logits, 1), lg)
    # max_new_tokens <= 2 (no graph) with processors
    for n in (1, 2):
        o = ours.generate(**kw, max_new_tokens=n, pad_token_id=0, return_dict_in_generate=True, output_scores=True, output_logits=True,
                          **opts)
        _teacher_forced(o, opts, ids.shape[1], n)


def test_errors(O, tiny):
    from audio_flamingo_b200 import AF3Error

    cfg, ours, _ = tiny
    feats, fmask, ids, am = _audio_inputs(O, cfg, [3.0], seed=6)
    kw = _kw(feats, fmask, ids, am)
    V = cfg.text_config.vocab_size
    for bad in (dict(bad_words_ids=[1, 2]), dict(bad_words_ids=[[1, -3]]), dict(sequence_bias={}), dict(sequence_bias={(V + 5,): 1.0}),
                dict(no_repeat_ngram_size=1.5), dict(forced_eos_token_id=-2)):
        from audio_flamingo_b200 import ops

        n0 = ops.LAUNCHES
        with pytest.raises(ValueError):
            ours.generate(**kw, max_new_tokens=4, **bad)
        assert ops.LAUNCHES == n0, f"{bad}: kernels were launched before the error"
    for bad in (dict(repetition_penalty=1.3), dict(do_sample=True), dict(num_beams=2), dict(exponential_decay_length_penalty=(2, 1.1)),
                dict(renormalize_logits=True), dict(remove_invalid_values=True), dict(logits_processor=[lambda i, s: s]),
                dict(prefix_allowed_tokens_fn=lambda b, i: [1]), dict(stop_strings=["x"])):
        with pytest.raises(AF3Error):
            ours.generate(**kw, max_new_tokens=4, **bad)
