"""Cost of the greedy logits processors (include/af3b200.h af3_logits_process_argmax) against the plain argmax, in one session:
  * kernels at B = 32, V = 152 064, history 780 + 128 tokens: af3_argmax alone, then the processor chain + selection with and
    without output_scores for several option mixes; CUDA-event time per launch over CUDA graphs of back-to-back launches
  * config 2 generate() (AF3-7B architecture, synthetic weights, batch 32 x 30 s clips, 128 greedy tokens): decode-step time with
    no_repeat_ngram_size=3 against no options, alternated; the no-option ids must equal a plain run's.
usage: python profiles/microbench_logits_processors.py [--skip-generate]"""
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from audio_flamingo_b200 import logits_process as LP  # noqa: E402
from audio_flamingo_b200 import ops  # noqa: E402

dev = "cuda"


def _graph_ms(fn, iters=50, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (iters * reps)


def kernels(B=32, V=152064, S=780, gen=128):
    rs = np.random.RandomState(0)
    logits = torch.from_numpy(rs.randn(B, V).astype(np.float32)).to(dev)
    Tmax = 1024
    prompt = torch.from_numpy(rs.randint(0, 151643, size=(B, Tmax)).astype(np.int64)).to(dev)
    generated = torch.from_numpy(rs.randint(0, 151643, size=(B, Tmax)).astype(np.int64)).to(dev)
    generated[:, 100:110] = generated[:, 20:30]        # repeats for the n-gram rule to find
    gen_idx = torch.full((1,), gen, dtype=torch.int32, device=dev)
    scores = torch.empty((B, V), device=dev)
    out = torch.empty((B,), dtype=torch.int64, device=dev)
    words = [[int(x) for x in rs.randint(0, 151643, size=n)] for n in (2, 2, 3, 3, 4)]
    mixes = {
        "3-gram": dict(no_repeat_ngram_size=3),
        "3-gram + 1000 suppressed + 5 multi-token bad words": dict(
            no_repeat_ngram_size=3, suppress_tokens=[int(x) for x in rs.choice(V, 1000, replace=False)], bad_words_ids=words),
        "all eight options": dict(
            no_repeat_ngram_size=3, suppress_tokens=[int(x) for x in rs.choice(V, 1000, replace=False)], bad_words_ids=words,
            sequence_bias={(5,): 1.5, (7, 9): -2.0, (1, 2, 3): 0.5}, min_length=S + 4, min_new_tokens=2, forced_eos_token_id=[151643],
            begin_suppress_tokens=[3, 4]),
    }
    base = _graph_ms(lambda: ops.argmax(logits, out=out))
    print(f"kernels at B={B}, V={V}, history {S} + {gen} (us per launch, graphs of 50 back-to-back launches x 20 replays)")
    print(f"  af3_argmax alone                                       : {base:7.2f}")
    for name, kw in mixes.items():
        opts = {k: kw.get(k) for k in LP.OPTIONS + ("forced_bos_token_id",)}
        c = LP.compile_processors(opts, [151643], S, S + 1000, V, Tmax)
        tables, static = torch.from_numpy(c.tables).to(dev), torch.from_numpy(c.static_add).to(dev)
        for sc in (None, scores):
            t = _graph_ms(lambda: ops.logits_process_argmax(logits, prompt, generated, gen_idx, tables, static, c.cap, out=out, scores=sc))
            print(f"  {name:<52} {'+ scores' if sc is not None else '        '}: {t:7.2f}  ({100 * (t / base - 1):+.1f} % vs argmax)")


def generate_config2(rounds=3):
    import bench
    from audio_flamingo_b200 import AF3FeatureExtractor, AudioFlamingo3ForConditionalGeneration

    cfg = bench.af3_config()
    m = AudioFlamingo3ForConditionalGeneration(cfg)
    m.to_empty(device=dev)
    m.to(torch.bfloat16)
    bench.init_synthetic_weights_(m, seed=0)
    B = bench.B_PER_GPU
    wave_np, ids_np = bench.synth_batch(B, seed=1000)
    wave, ids = torch.from_numpy(wave_np).to(dev), torch.from_numpy(ids_np).to(dev)
    fe = AF3FeatureExtractor(dev)
    feats = fe.from_device_waveform(wave, [wave_np.shape[1]] * B)
    kw = dict(input_ids=ids, attention_mask=torch.ones_like(ids), input_features=feats["input_features"],
              input_features_mask=feats["input_features_mask"], max_new_tokens=bench.NEW_TOKENS, do_sample=False)
    print(f"config 2 generate(): batch {B}, prompt {ids.shape[1]}, {bench.NEW_TOKENS} new tokens")
    plain = m.generate(**kw)
    m.generate(**kw, no_repeat_ngram_size=3)
    torch.cuda.synchronize()
    steps = {"none": [], "3-gram": []}
    for r in range(rounds):
        for tag, extra in (("none", {}), ("3-gram", dict(no_repeat_ngram_size=3))):
            m.stage_events = []
            out = m.generate(**kw, **extra)
            torch.cuda.synchronize()
            ev = dict(m.stage_events)
            m.stage_events = None
            step = ev["prefill_done"].elapsed_time(ev["decode_done"]) / (bench.NEW_TOKENS - 1)
            steps[tag].append(step)
            print(f"  round {r} {tag:>6}: decode step {step:6.3f} ms")
            if tag == "none":
                assert torch.equal(out, plain), "no-option ids differ from the plain run"
    a, b = np.median(steps["none"]), np.median(steps["3-gram"])
    print(f"  median decode step: no options {a:.3f} ms, no_repeat_ngram_size=3 {b:.3f} ms ({100 * (b / a - 1):+.2f} %); "
          "no-option ids == plain run")


if __name__ == "__main__":
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {smi.stdout.strip()}")
    kernels()
    if "--skip-generate" not in sys.argv:
        generate_config2()
