"""Few-token (decode) GEMM: time per launch and its split into weight streaming vs reduction/epilogue tail, as a function of the
number of K splits, whose partial tiles are reduced through global memory (the split-K tail: last accumulator ready -> last CTA
exit); this sweep measures (a) how the tail scales with the split count and (b) whether fewer CTAs still pull the weights at HBM
speed.
    python profiles/microbench_splitk.py > splitk.json
us per launch: CUDA events around a graph of 48 back-to-back launches (no PDL), weights rotated over 12 copies so every launch
streams from HBM.  stream / tail: library trace (%globaltimer) of 12 eager launches, medians."""
import json
import os
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from audio_flamingo_b200 import _lib, ops  # noqa: E402

torch.manual_seed(0)
dev = "cuda"
M = 32
lib = _lib.load()
slot_words = lib.af3_trace_slot_bytes() // 8


def run_shape(name, N, K, mode, copies=12, iters=48):
    ws = [(torch.randn(N, K, device=dev) * 0.02).to(torch.bfloat16) for _ in range(copies)]
    x = torch.randn(M, K, device=dev).to(torch.bfloat16)
    bias = torch.zeros(N, device=dev, dtype=torch.bfloat16)
    out = torch.randn(M, N, device=dev).to(torch.bfloat16)

    def run(i):
        w = ws[i % copies]
        if mode == "bias":
            ops.linear(x, w, bias, out=out)
        else:
            ops.linear(x, w, resid=out, out=out)

    rows = []
    for ks in (1, 2, 3, 4, 5, 6, 8):
        os.environ["AF3_KSPLIT"] = str(ks)
        for i in range(4):
            run(i)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(iters):
                run(i)
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / iters
        # stream / tail from the trace
        n_tr = 12
        buf = torch.zeros((n_tr * slot_words,), device=dev, dtype=torch.int64)
        lib.af3_trace_begin(buf.data_ptr(), buf.numel() * 8)
        for i in range(n_tr):
            run(i)
        torch.cuda.synchronize()
        lib.af3_trace_end()
        raw = buf.view(n_tr, -1, 4).cpu()
        stream, tail, ctas = [], [], 0
        for s in range(2, n_tr):
            m = raw[s]
            live = m[:, 0] > 0
            ctas = int(live.sum())
            t_wait = int(m[live, 1][m[live, 1] > 0].min())
            stream.append((int(m[live, 2].max()) - t_wait) / 1e3)
            tail.append((int(m[live, 3].max()) - int(m[live, 2].max())) / 1e3)
        rows.append({"k_splits_requested": ks, "ctas": ctas, "us_per_launch": round(us, 2), "tbs": round(N * K * 2 / us / 1e6, 2),
                     "stream_us_median": round(statistics.median(stream), 2), "tail_us_median": round(statistics.median(tail), 2)})
        del g
    os.environ.pop("AF3_KSPLIT", None)
    return {"shape": name, "n_feat": N, "K": K, "epilogue": mode, "weight_bytes": N * K * 2, "ideal_us_at_3350_gbs": round(N * K * 2 / 3350e3, 2),   # H100 SXM data-sheet HBM3 bandwidth
            "sweep": rows}


res = [run_shape("qkv", 4608, 3584, "bias"), run_shape("o_proj", 3584, 3584, "resid"), run_shape("down", 3584, 18944, "resid")]
print(json.dumps({"what": __doc__.split("\n")[0], "results": res}, indent=1))
