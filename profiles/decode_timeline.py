#!/usr/bin/env python
"""In-graph timeline of one decode step (programmatic dependent launch ON, nothing serialised).

Nsight Compute replays kernels one at a time, so it cannot show where the decode step's slack sits.  This tool opens the library's trace (include/af3b200.h: af3_trace_begin), runs
generate() at the bench's shape (AF3-7B decoder, 32 sequences, 780-token prompts) so that the decode step is captured
in a CUDA graph WITH the trace slots baked in, replays it, and reads back per-CTA %globaltimer stamps of the LAST replay:
    mark 0 kernel entry, 1 after griddepcontrol.wait, 2 main loop done (GEMM: last accumulator ready), 3 exit.
Output: JSON (one record per launch + per-kind aggregates) and a markdown summary.

    python profiles/decode_timeline.py --out /tmp/decode_timeline --tag base
Environment knobs under test are simply inherited (AF3_PDL, AF3_KSPLIT, ...).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(Path(tempfile.gettempdir()) / "decode_timeline"))
    ap.add_argument("--tag", default="default")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--prompt", type=int, default=780)
    ap.add_argument("--new-tokens", type=int, default=24)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--fp8", action="store_true", help="FP8 decoder projections (load_reference_state_dict(quantization='fp8'))")
    args = ap.parse_args()

    import bench
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    cfg = bench.af3_config()
    cfg.text_config.num_hidden_layers = args.layers
    cfg.audio_config.num_hidden_layers = 1  # the audio tower is not exercised here (text-only prompts)
    model = AudioFlamingo3ForConditionalGeneration(cfg)
    model.to_empty(device=dev)
    model.to(torch.bfloat16)
    bench.init_synthetic_weights_(model, seed=0)
    if args.fp8:
        model.load_reference_state_dict(model.state_dict(), device=dev, quantization="fp8")
    rs = np.random.RandomState(0)
    ids = torch.from_numpy(rs.randint(1, 151643, size=(args.batch, args.prompt)).astype(np.int64)).to(dev)
    am = torch.ones_like(ids)

    from audio_flamingo_b200.trace import DecodeTrace

    # warm run without tracing (configures kernels, allocator), state dropped so the traced run captures a fresh graph
    model.generate(input_ids=ids, attention_mask=am, max_new_tokens=4)
    model.release_decode_state()
    torch.cuda.synchronize()

    model.stage_events = []
    with DecodeTrace(dev) as tr:
        model.generate(input_ids=ids, attention_mask=am, max_new_tokens=args.new_tokens)
    n_rec = tr.n_recorded
    ev = dict(model.stage_events)
    decode_ms = ev["prefill_done"].elapsed_time(ev["decode_done"])
    model.stage_events = None
    launches = tr.graph_launches()
    assert launches, "the decode step was not captured (max_new_tokens too small?)"
    model.release_decode_state()   # the captured graph writes into tr.buf: drop it before the buffer goes away
    step_us = max(r["exit_max"] for r in launches if r["exit_max"] is not None) - launches[0]["entry_min"]
    agg = DecodeTrace.aggregate(launches)

    out = {"tag": args.tag, "env": {k: v for k, v in os.environ.items() if k.startswith("AF3_")},
           "shape": {"batch": args.batch, "prompt": args.prompt, "layers": args.layers, "new_tokens": args.new_tokens},
           "decode_ms_per_step_events": decode_ms / (args.new_tokens - 1), "step_us_from_trace": step_us,
           "launches_in_graph": len(launches), "slots_recorded": n_rec, "per_kind": agg, "launches": launches}
    base = f"{args.out}_{args.tag}"
    Path(base + ".json").write_text(json.dumps(out))
    lines = [f"# decode-step timeline ({args.tag}): {step_us:.1f} us per step from the trace, "
             f"{decode_ms / (args.new_tokens - 1) * 1e3:.1f} us per step by CUDA events over the decode stage", "",
             f"env: {out['env']}", "",
             "Sums over the launches of one step, in us.  slot = last exit - predecessor's last exit (exclusive share of the step; the slots add up "
             "to the step); body = dependency resolved -> last exit; stream = -> last accumulator ready; tail = rest of the body; resident "
             "before dep. = time the kernel sat resident ahead of its dependency (pre-wait weight prefetch window); gap = predecessor's last "
             "exit -> dependency resolved.", "",
             "| kernel | launches | slot | body | stream | tail | resident before dep. | gap after predecessor |",
             "|---|---|---|---|---|---|---|---|"]
    for name, a in sorted(agg.items(), key=lambda kv: -kv[1]["slot_us"]):
        lines.append(f"| {name} | {a['n']} | {a['slot_us']:.1f} | {a['body_us']:.1f} | {a['stream_us']:.1f} | {a['tail_us']:.1f} | {a['lead_us']:.1f} | {a['gap_us']:.1f} |")
    lines += ["", "First layer in launch order (us since step start):", "",
              "| kernel | ctas | entry min..max | dep. resolved min..max | main loop done | exit min..max |", "|---|---|---|---|---|---|"]
    for r in launches[:12]:
        f = lambda v: "-" if v is None else f"{v:.1f}"  # noqa: E731
        lines.append(f"| {r['kind']} | {r['ctas']} | {f(r['entry_min'])}..{f(r['entry_max'])} | {f(r['wait_min'])}..{f(r['wait_max'])} | "
                     f"{f(r['mid_max'])} | {f(r['exit_min'])}..{f(r['exit_max'])} |")
    Path(base + ".md").write_text("\n".join(lines) + "\n")
    quant_us = sum(v["slot_us"] for k, v in agg.items() if k.startswith("quant_fp8"))
    out["quant_fp8_share"] = quant_us / step_us
    print(json.dumps({k: out[k] for k in ("tag", "decode_ms_per_step_events", "step_us_from_trace", "launches_in_graph", "quant_fp8_share")}))


if __name__ == "__main__":
    main()
