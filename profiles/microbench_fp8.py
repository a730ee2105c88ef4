"""bf16 against FP8 decoder projections in one session, alternating: the four decode-shape GEMMs at 32 tokens (rotating weight
copies, so every launch streams its weights from HBM), the four prefill shapes at 24 960 tokens (FP8 time includes the
activation quantization, reported beside it), and config 2 generate() (AF3-7B architecture, synthetic weights, batch 32 x 30 s
clips, 128 greedy tokens): decode-step ms, prefill ms, generated tokens/s and the share of greedy ids FP8 and bf16 agree on.
usage: python profiles/microbench_fp8.py [--skip-generate]"""
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from audio_flamingo_b200 import ops  # noqa: E402
from audio_flamingo_b200.modeling import quantize_fp8_blocks  # noqa: E402

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


def _graph_ms(fn, iters):
    for i in range(3):
        fn(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(iters):
            fn(i)
    g.replay()
    torch.cuda.synchronize()
    return _events_ms(lambda i: g.replay(), 1) / iters


def gemm_fns(rows, K, epi, M, copies):
    n = rows // 2 if epi == "swiglu" else rows
    wb = [(torch.randn(rows, K, device=dev) * 0.02).to(torch.bfloat16) for _ in range(copies)]
    wf = [quantize_fp8_blocks(w) for w in wb]
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

    def quant(i):
        return ops.quant_fp8(x)

    xq = quant(0)

    def f8(i, with_quant=True):
        q = quant(i) if with_quant else xq
        w, s = wf[i % copies]
        if epi == "swiglu":
            ops.swiglu_linear_fp8(q, w, s, n, out=out)
        elif epi == "bias":
            ops.linear_fp8(q, w, s, bias, out=out)
        else:
            ops.linear_fp8(q, w, s, resid=out, out=out)

    return bf, f8, quant, wb[0].numel()


def decode_gemms(rounds=3):
    print("decode GEMMs, 32 tokens (us per launch; weight TB/s; FP8 includes its quant launch)")
    for name, rows, K, epi in SHAPES:
        bf, f8, quant, numel = gemm_fns(rows, K, epi, 32, copies=12 if rows * K < 1e8 else 6)
        for r in range(rounds):
            tb = _graph_ms(bf, 48) * 1e3
            tf = _graph_ms(f8, 48) * 1e3
            tq = _graph_ms(quant, 48) * 1e3
            print(f"  {name:8s} round {r}: bf16 {tb:7.2f} us {numel * 2 / tb / 1e6:5.2f} TB/s | fp8 {tf:7.2f} us "
                  f"{numel / tf / 1e6:5.2f} TB/s (quant {tq:5.2f} us)")


def prefill_gemms(M=24960, rounds=2):
    print(f"prefill GEMMs, {M} tokens (TFLOP/s; FP8 time includes the quant kernel, whose time is shown)")
    for name, rows, K, epi in SHAPES:
        bf, f8, quant, _ = gemm_fns(rows, K, epi, M, copies=1)
        flop = 2.0 * M * rows * K
        for r in range(rounds):
            tb = _events_ms(bf, 5)
            tf = _events_ms(f8, 5)
            tq = _events_ms(quant, 5)
            print(f"  {name:8s} round {r}: bf16 {tb:7.3f} ms {flop / tb / 1e9:6.1f} TFLOP/s | fp8 {tf:7.3f} ms "
                  f"{flop / tf / 1e9:6.1f} TFLOP/s (quant {tq:6.3f} ms)")


def generate_config2(rounds=2):
    import bench
    from audio_flamingo_b200 import AF3FeatureExtractor, AudioFlamingo3ForConditionalGeneration

    cfg = bench.af3_config()
    mb = AudioFlamingo3ForConditionalGeneration(cfg)
    mb.to_empty(device=dev)
    mb.to(torch.bfloat16)
    bench.init_synthetic_weights_(mb, seed=0)
    mf = AudioFlamingo3ForConditionalGeneration(cfg)
    mf.load_reference_state_dict(mb.state_dict(), device=dev, quantization="fp8")
    B = bench.B_PER_GPU
    wave_np, ids_np = bench.synth_batch(B, seed=1000)
    wave, ids = torch.from_numpy(wave_np).to(dev), torch.from_numpy(ids_np).to(dev)
    fe = AF3FeatureExtractor(dev)
    feats = fe.from_device_waveform(wave, [wave_np.shape[1]] * B)
    kw = dict(input_ids=ids, attention_mask=torch.ones_like(ids), input_features=feats["input_features"],
              input_features_mask=feats["input_features_mask"], max_new_tokens=bench.NEW_TOKENS, do_sample=False)
    print(f"config 2 generate(): batch {B}, prompt {ids.shape[1]}, {bench.NEW_TOKENS} new tokens")
    outs = {}
    for m in (mb, mf):
        m.generate(**kw)  # capture the decode graph, warm the allocator
    torch.cuda.synchronize()
    for r in range(rounds):
        for tag, m in (("bf16", mb), ("fp8", mf)):
            m.stage_events = []
            t = _events_ms(lambda i: outs.__setitem__(tag, m.generate(**kw)), 1)
            ev = dict(m.stage_events)
            m.stage_events = None
            prefill = ev["audio_done"].elapsed_time(ev["prefill_done"])
            decode = ev["prefill_done"].elapsed_time(ev["decode_done"])
            print(f"  round {r} {tag}: {t:8.1f} ms, prefill {prefill:7.1f} ms, decode step {decode / (bench.NEW_TOKENS - 1):6.3f} ms, "
                  f"{B * bench.NEW_TOKENS / t * 1e3:7.1f} generated tokens/s")
    S = ids.shape[1]
    agree = (outs["bf16"][:, S:] == outs["fp8"][:, S:]).float().mean().item()
    print(f"  greedy ids FP8 == bf16: {100 * agree:.1f} % of generated tokens")


if __name__ == "__main__":
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"GPU: {smi.stdout.strip()}")
    decode_gemms()
    prefill_gemms()
    if "--skip-generate" not in sys.argv:
        generate_config2()
