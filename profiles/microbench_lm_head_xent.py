"""Cost of the teacher-forced loss (include/af3b200.h af3_lm_head_xent) at config 2's LM-head shape, in one session:
  * T = 24 960 tokens (32 x 780), V = 152 064, K = 3 584 (27.2 TFLOP): the present head ops.linear(out_f32=True), the fused
    loss-only launch and the fused launch that also stores the logits; CUDA-event time per launch over CUDA graphs of
    back-to-back launches, the variants alternated; their token_nll must be bit-identical
  * the merge and totals kernels alone, from a torch.profiler run of its own
  * peak memory growth of forward(labels, logits_to_keep=1) against forward(labels) on the AF3-7B decoder geometry with two layers
    (synthetic weights): 32 x 780 tokens and one 15 000-token prompt (20 windows of audio)
usage: python profiles/microbench_lm_head_xent.py [--skip-memory]"""
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from audio_flamingo_b200 import ops  # noqa: E402

dev = "cuda"
bf16 = torch.bfloat16


def _graph(fn, iters):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def _time(g):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def kernels(T=24960, V=152064, K=3584, iters=5, reps=6):
    g = torch.Generator(device=dev).manual_seed(0)
    x = (torch.randn(T, K, device=dev, generator=g) * 0.5).to(bf16)
    w = (torch.randn(V, K, device=dev, generator=g) * (2.0 / K ** 0.5)).to(bf16)
    lab = torch.randint(0, V, (T,), device=dev, generator=g)
    out = torch.empty((T, V), device=dev)
    res = {}
    variants = {
        "present head (ops.linear out_f32)": lambda: ops.linear(x, w, out=out, out_f32=True),
        "fused loss only": lambda: res.__setitem__("loss_only", ops.lm_head_xent(x, w, lab)[1]),
        "fused loss + logits": lambda: res.__setitem__("with_logits", ops.lm_head_xent(x, w, lab, store_logits=True)[1]),
    }
    graphs = {k: _graph(f, iters) for k, f in variants.items()}
    times = {k: [] for k in variants}
    for _ in range(reps):
        for k, gr in graphs.items():
            times[k].append(_time(gr) / iters)
    flop = 2.0 * T * V * K
    rows = {}
    for k, ts in times.items():
        ms = sorted(ts)[len(ts) // 2]
        rows[k] = {"ms_median": round(ms, 3), "ms_min": round(min(ts), 3), "ms_max": round(max(ts), 3), "TFLOP/s": round(flop / ms / 1e9, 1)}
        print(f"{k:36s} {ms:8.3f} ms (min {min(ts):.3f}, max {max(ts):.3f})  {flop / ms / 1e9:6.1f} TFLOP/s")
    same = torch.equal(res["loss_only"], res["with_logits"])
    print("token_nll loss-only == with logits:", same)
    base = rows["present head (ops.linear out_f32)"]["ms_median"]
    print(f"loss-only / present head: {rows['fused loss only']['ms_median'] / base:.3f}")

    # merge + totals kernels: a profiler run of its own
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            ops.lm_head_xent(x, w, lab)
        torch.cuda.synchronize()
    merge = {}
    for ev in prof.key_averages():
        if "xent_merge_kernel" in ev.key or "xent_totals_kernel" in ev.key or "gemm_tok_kernel" in ev.key:
            t = getattr(ev, "device_time_total", None) or ev.cuda_time_total
            merge[ev.key.split("(")[0]] = round(t / ev.count, 1)
    print("per-launch kernel time, us:", merge)
    del out
    torch.cuda.empty_cache()
    return {"rows": rows, "bit_identical": same, "kernel_us": merge, "scratch_MB": ops._lib.load().af3_lm_head_xent_scratch_bytes(T, V) / 1e6}


def memory():
    """Peak growth of forward(labels) with logits_to_keep = 1 and 0 on the AF3-7B decoder geometry (2 layers, synthetic)."""
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration
    from oracle import af3_oracle as O

    m = AudioFlamingo3ForConditionalGeneration(O.hf_config("mid"))
    m.to_empty(device=dev)
    m.to(bf16)
    g = torch.Generator(device=dev).manual_seed(1)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02, generator=g)
        for l in m.language_model.model.layers:
            l.input_layernorm.weight.fill_(1)
            l.post_attention_layernorm.weight.fill_(1)
        m.language_model.model.norm.weight.fill_(1)
    V = m.vocab_size
    out = {}
    for name, (B, S) in {"32 x 780": (32, 780), "1 x 15000 (20 windows)": (1, 15000)}.items():
        emb = (torch.randn(B, S, m.config.text_config.hidden_size, device=dev, generator=g) * 0.02).to(bf16)
        lab = torch.randint(0, V, (B, S), device=dev, generator=g)
        row = {}
        for keep in (1, 0):
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            r = m(inputs_embeds=emb, labels=lab, logits_to_keep=keep)
            torch.cuda.synchronize()
            row[f"logits_to_keep={keep}"] = round((torch.cuda.max_memory_allocated() - base) / 2**30, 3)
            row[f"loss (keep={keep})"] = r.loss.item()
            del r
        row["B*S*V*4 GiB"] = round(B * S * V * 4 / 2**30, 3)
        print(name, row)
        out[name] = row
    return out


if __name__ == "__main__":
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("GPU:", smi)
    result = {"gpu": smi, "kernels": kernels()}
    if "--skip-memory" not in sys.argv:
        result["memory_GiB"] = memory()
    print(json.dumps(result))
