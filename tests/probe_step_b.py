"""Times a few eager Step-B steps at batch 16 (no profiler): python tests/probe_step_b.py [steps]"""
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from objgan_b200 import synth, trainer

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 4
random.seed(1234)
tr = trainer.StepBTrainer(device="cuda", seed=1234)
host = trainer.pin(synth.make_inputs(16, seed=1234, parity=False))
host.pop("eps")
dev = tr.to_device(host)
for i in range(2):
    tr.step(dev)
    torch.cuda.synchronize()
    print("warm-up step", i, "done", flush=True)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
t0 = time.perf_counter()
e0.record()
for _ in range(steps):
    tr.step(dev)
e1.record()
t_enq = (time.perf_counter() - t0) / steps
torch.cuda.synchronize()
print(f"step b B=16: host enqueue {t_enq * 1e3:.1f} ms/step, "
      f"GPU {e0.elapsed_time(e1) / steps:.1f} ms/step, peak memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB", flush=True)
