"""Times a few eager Step-A steps at batch 16 with progress lines (no profiler): python tests/probe_step_a.py [steps]"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from objgan_b200 import synth, trainer

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 4
tr = trainer.StepATrainer(device="cuda", seed=1234)
host = trainer.pin(synth.make_inputs(16, seed=1234, parity=False))
host.pop("eps")
dev = tr.to_device(host)
for i in range(2):
    t0 = time.perf_counter()
    tr.step(dev)
    torch.cuda.synchronize()
    print(f"warm-up step {i}: {time.perf_counter() - t0:.2f} s", flush=True)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(steps):
    tr.step(dev)
e1.record()
torch.cuda.synchronize()
print(f"step a B=16: GPU {e0.elapsed_time(e1) / steps:.1f} ms/step", flush=True)
