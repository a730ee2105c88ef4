"""Runner for Nsight Compute passes: builds the bench workload,
runs warm-up steps unprofiled, then ONE step between cudaProfilerStart/Stop.
  launch list : ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none -c 1600 --csv --log-file X python profiles/ncu_driver.py
  top kernel  : ncu --profile-from-start off --set full --clock-control none --import-source on -k regex:gemm_kernel -c 3 -o X python profiles/ncu_driver.py
Decode steps are limited (AF3_NCU_NEW_TOKENS, default 3) so the profiled region stays short; eager decode unless
AF3_NCU_GRAPH=1 (then ncu --graph-profiling node times the kernel nodes of the replayed decode graph)."""
import os
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402

from audio_flamingo_b200 import AF3FeatureExtractor, AudioFlamingo3ForConditionalGeneration  # noqa: E402

new = int(os.environ.get("AF3_NCU_NEW_TOKENS", "3"))
dev = torch.device("cuda", 0)
model = AudioFlamingo3ForConditionalGeneration(bench.af3_config())
model.to_empty(device=dev)
model.to(torch.bfloat16)
bench.init_synthetic_weights_(model, seed=0)
fe = AF3FeatureExtractor(dev)
wave_np, ids_np = bench.synth_batch(bench.B_PER_GPU, seed=1000)
wave, ids = torch.from_numpy(wave_np).to(dev), torch.from_numpy(ids_np).to(dev)
mask = torch.ones_like(ids)


def step():
    feats = fe.from_device_waveform(wave, [wave_np.shape[1]] * bench.B_PER_GPU)
    return model.generate(input_ids=ids, attention_mask=mask, input_features=feats["input_features"],
                          input_features_mask=feats["input_features_mask"], max_new_tokens=new,
                          use_cuda_graph=os.environ.get("AF3_NCU_GRAPH", "0") == "1")


step()
torch.cuda.synchronize()
torch.cuda.profiler.start()
step()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("profiled one step")
