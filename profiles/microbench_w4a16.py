"""bf16, FP8 and W4A16 decoder projections in one session, alternating: the four decode-shape GEMMs at 32 tokens (CUDA graphs of
back-to-back launches over rotating weight copies, so every launch streams its weights from HBM; FP8 includes its activation
quantization), the cost of af3_dequant_w4a16 per layer, and config 2 (AF3-7B architecture, synthetic weights, batch 32 x 30 s
clips, 128 greedy tokens): prefill ms, ms per decode step, generated tokens/s and the memory each model holds after loading.
usage: python profiles/microbench_w4a16.py [--skip-generate]"""
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from audio_flamingo_b200 import ops  # noqa: E402
from audio_flamingo_b200.modeling import quantize_fp8_blocks, quantize_w4a16  # noqa: E402

dev = "cuda"
torch.manual_seed(0)
# (name, weight rows, K, epilogue) of one Qwen2.5-7B decoder layer
SHAPES = [("qkv", 4608, 3584, "bias"), ("o_proj", 3584, 3584, "resid"), ("gate_up", 2 * 18944, 3584, "swiglu"), ("down", 3584, 18944, "resid")]


def _events_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _graph(fn, iters):
    for i in range(3):
        fn(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(iters):
            fn(i)
    g.replay()
    torch.cuda.synchronize()
    return lambda: _events_ms(lambda i: g.replay(), 1) / iters


def gemm_fns(rows, K, epi, M, copies):
    n = rows // 2 if epi == "swiglu" else rows
    wb = [(torch.randn(rows, K, device=dev) * 0.02).to(torch.bfloat16) for _ in range(copies)]
    wf = [quantize_fp8_blocks(w) for w in wb]
    w4 = [quantize_w4a16(w) for w in wb]
    x = torch.randn(M, K, device=dev).to(torch.bfloat16)
    bias = torch.zeros(n, device=dev, dtype=torch.bfloat16)
    out = torch.randn(M, n, device=dev).to(torch.bfloat16)

    def bf(i):
        w = wb[i % copies]
        if epi == "swiglu":
            ops.swiglu_linear(x, w, n, out=out, concat=True)
        elif epi == "bias":
            ops.linear(x, w, bias, out=out)
        else:
            ops.linear(x, w, resid=out, out=out)

    def f8(i):
        q = ops.quant_fp8(x)
        w, s = wf[i % copies]
        if epi == "swiglu":
            ops.swiglu_linear_fp8(q, w, s, n, out=out)
        elif epi == "bias":
            ops.linear_fp8(q, w, s, bias, out=out)
        else:
            ops.linear_fp8(q, w, s, resid=out, out=out)

    def q4(i):
        p, s = w4[i % copies]
        if epi == "swiglu":
            ops.swiglu_linear_w4a16(x, p, s, n, out=out)
        elif epi == "bias":
            ops.linear_w4a16(x, p, s, bias, out=out)
        else:
            ops.linear_w4a16(x, p, s, resid=out, out=out)

    return dict(bf16=bf, fp8=f8, w4a16=q4), rows * K


def decode_gemms(rounds=3):
    print(f"decode GEMMs, 32 tokens, CUDA graphs of 48 launches, {rounds} alternated rounds: median [min, max] us per launch, "
          "weight bytes / median time (FP8 includes its activation quant launch; W4A16 bytes include the bf16 scales)")
    for name, rows, K, epi in SHAPES:
        fns, numel = gemm_fns(rows, K, epi, 32, copies=12 if rows * K < 1e8 else 6)
        wbytes = dict(bf16=2 * numel, fp8=numel + numel // (128 * 128) * 4, w4a16=numel // 2 + numel // 128 * 2)
        graphs = {k: _graph(f, 48) for k, f in fns.items()}
        t = {k: [] for k in fns}
        for _ in range(rounds):
            for k, g in graphs.items():
                t[k].append(g() * 1e3)
        line = []
        for k, v in t.items():
            med = statistics.median(v)
            line.append(f"{k} {med:7.2f} [{min(v):7.2f}, {max(v):7.2f}] us {wbytes[k] / med / 1e6:5.2f} TB/s")
        print(f"  {name:8s} " + " | ".join(line))
        del graphs, fns
        torch.cuda.empty_cache()


def dequant_cost(rounds=3):
    print("af3_dequant_w4a16 of one decoder layer's four projections (ms)")
    ws = [quantize_w4a16((torch.randn(rows, K, device=dev) * 0.02).to(torch.bfloat16)) for _, rows, K, _ in SHAPES]
    scratch = torch.empty((max(p.shape[0] * p.shape[1] * 8 for p, _ in ws),), device=dev, dtype=torch.bfloat16)
    for r in range(rounds):
        t = _events_ms(lambda i: [ops.dequant_w4a16(p, s, out=scratch) for p, s in ws], 10)
        print(f"  round {r}: {t:.3f} ms per layer, {28 * t:.2f} ms for 28 layers")


def generate_config2(rounds=3):
    import bench
    from audio_flamingo_b200 import AF3FeatureExtractor, AudioFlamingo3ForConditionalGeneration

    cfg = bench.af3_config()
    models, mem = {}, {}
    sd = None
    for tag, q in (("bf16", None), ("fp8", "fp8"), ("w4a16", "w4a16")):
        torch.cuda.synchronize()
        a0 = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        m = AudioFlamingo3ForConditionalGeneration(cfg)
        if q is None:
            m.to_empty(device=dev)
            m.to(torch.bfloat16)
            bench.init_synthetic_weights_(m, seed=0)
            sd = m.state_dict()
        else:
            m.load_reference_state_dict(sd, device=dev, quantization=q)
        m.language_model._check_ready()  # packed weights (W4A16: and its dequantization scratch)
        torch.cuda.synchronize()
        mem[tag] = (torch.cuda.memory_allocated() - a0, torch.cuda.max_memory_allocated() - a0)
        models[tag] = m
    print("memory of each model after loading (torch.cuda.memory_allocated delta; peak during the load), GB: "
          + ", ".join(f"{k} {v[0] / 1e9:.2f} (peak {v[1] / 1e9:.2f})" for k, v in mem.items()))
    del sd
    B = bench.B_PER_GPU
    wave_np, ids_np = bench.synth_batch(B, seed=1000)
    wave, ids = torch.from_numpy(wave_np).to(dev), torch.from_numpy(ids_np).to(dev)
    fe = AF3FeatureExtractor(dev)
    feats = fe.from_device_waveform(wave, [wave_np.shape[1]] * B)
    kw = dict(input_ids=ids, attention_mask=torch.ones_like(ids), input_features=feats["input_features"],
              input_features_mask=feats["input_features_mask"], max_new_tokens=bench.NEW_TOKENS, do_sample=False)
    print(f"config 2 generate(): batch {B}, prompt {ids.shape[1]}, {bench.NEW_TOKENS} new tokens, {rounds} alternated rounds")
    outs, res = {}, {k: [] for k in models}
    for m in models.values():
        m.generate(**kw)  # capture the decode graph, warm the allocator
    torch.cuda.synchronize()
    for r in range(rounds):
        for tag, m in models.items():
            m.stage_events = []
            t = _events_ms(lambda i: outs.__setitem__(tag, m.generate(**kw)), 1)
            ev = dict(m.stage_events)
            m.stage_events = None
            prefill = ev["audio_done"].elapsed_time(ev["prefill_done"])
            step = ev["prefill_done"].elapsed_time(ev["decode_done"]) / (bench.NEW_TOKENS - 1)
            res[tag].append((t, prefill, step))
            print(f"  round {r} {tag:5s}: {t:8.1f} ms, prefill {prefill:7.1f} ms, decode step {step:6.3f} ms, "
                  f"{B * bench.NEW_TOKENS / t * 1e3:7.1f} generated tokens/s")
    for tag, v in res.items():
        steps, pre = [x[2] for x in v], [x[1] for x in v]
        print(f"  {tag:5s}: decode step median {statistics.median(steps):.3f} ms [{min(steps):.3f}, {max(steps):.3f}], "
              f"prefill median {statistics.median(pre):.1f} ms [{min(pre):.1f}, {max(pre):.1f}]")
    S = ids.shape[1]
    for tag in ("fp8", "w4a16"):
        agree = (outs["bf16"][:, S:] == outs[tag][:, S:]).float().mean().item()
        print(f"  greedy ids {tag} == bf16: {100 * agree:.1f} % of generated tokens")


if __name__ == "__main__":
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {smi.stdout.strip()}")
    decode_gemms()
    dequant_cost()
    if "--skip-generate" not in sys.argv:
        generate_config2()
