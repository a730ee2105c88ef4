"""Normal-mode (token-major) GEMM at every shape config 2 runs through it, full size, each with its real epilogue.
    python profiles/microbench_prefill_gemm.py > prefill_gemm.json
Per shape: ms per launch (CUDA events around a captured graph of back-to-back launches, median of 3 replays), TFLOP/s from the
shape (2 M N K; SwiGLU: N = both halves), and the SHA-256 of the output of one launch on seeded inputs, so that two builds can
be compared output for output.  The first line names the card, its power limit and max SM clock."""
import hashlib
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from audio_flamingo_b200 import ops  # noqa: E402

dev = "cuda"
bf16 = torch.bfloat16

# name, M (tokens), N (output features; SwiGLU: intermediate size), K, epilogue
SHAPES = [
    ("enc.qkv", 48000, 3840, 1280, "bias"),
    ("enc.out_proj", 48000, 1280, 1280, "bias+resid_inplace"),
    ("enc.fc1", 48000, 5120, 1280, "bias+gelu"),
    ("enc.fc2", 48000, 1280, 5120, "bias+resid_inplace"),
    ("conv1", 96000, 1280, 384, "bias+gelu"),
    ("conv2", 48000, 1280, 3840, "bias+gelu+pos"),
    ("proj.linear_1", 24000, 3584, 1280, "bias+gelu"),
    ("proj.linear_2", 24000, 3584, 3584, "bias"),
    ("prefill.qkv", 24960, 4608, 3584, "bias"),
    ("prefill.o_proj", 24960, 3584, 3584, "resid_inplace"),
    ("prefill.gate_up", 24960, 18944, 3584, "swiglu_concat"),
    ("prefill.down", 24960, 3584, 18944, "resid_inplace"),
]
POS_PERIOD = 1500  # encoder positions per window (conv2's positional-embedding add)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else None}


def make(name, M, N, K, epi, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, device=dev, generator=g) * scale).to(bf16)  # noqa: E731
    x = rnd(M, K)
    wscale = K ** -0.5
    if epi == "swiglu_concat":
        w = rnd(2 * N, K, scale=wscale)
        out = torch.empty(M, N, device=dev, dtype=bf16)
        return lambda: ops.swiglu_linear(x, w, N, out=out, concat=True), out, None, None
    w = rnd(N, K, scale=wscale)
    bias = rnd(N, scale=0.5) if "bias" in epi else None
    gelu = "gelu" in epi
    if epi.endswith("resid_inplace"):
        out = rnd(M, N)
        resid0 = out.clone()
        return lambda: ops.linear(x, w, bias, gelu=gelu, resid=out, out=out), out, resid0, out
    out = torch.empty(M, N, device=dev, dtype=bf16)
    if epi.endswith("pos"):
        pos = rnd(POS_PERIOD, N)
        return lambda: ops.linear(x, w, bias, gelu=gelu, resid=pos, res_period=POS_PERIOD, out=out), out, None, None
    return lambda: ops.linear(x, w, bias, gelu=gelu, out=out), out, None, None


def run_shape(i, name, M, N, K, epi, iters=10, replays=3):
    fn, out, resid0, inplace = make(name, M, N, K, epi, seed=1000 + i)
    fn()  # first launch on the seeded inputs: this output is hashed
    torch.cuda.synchronize()
    digest = hashlib.sha256(out.view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(iters):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    ms = []
    for _ in range(replays):
        if inplace is not None:  # keep the in-place accumulator bounded
            inplace.copy_(resid0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / iters)
    n_mma = 2 * N if epi.startswith("swiglu") else N
    t = statistics.median(ms)
    return {"name": name, "M": M, "N": n_mma, "K": K, "epilogue": epi, "ms": round(t, 4),
            "tflops": round(2.0 * M * n_mma * K / (t * 1e-3) / 1e12, 1), "ms_all": [round(v, 4) for v in ms], "sha256": digest}


def main():
    assert torch.cuda.is_available(), "needs a GPU"
    print(json.dumps({"card": card()}), flush=True)
    for i, s in enumerate(SHAPES):
        print(json.dumps(run_shape(i, *s)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
