"""Per-kernel time breakdown of one eager ResNet-50 training step (torch.profiler / CUPTI), written to
profiles/step_profile.txt and profiles/step_kernels.txt (generated output, not tracked).  Used to decide what to
optimise next."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

from b200ddl import optim
from b200ddl.models.resnet_engine import EngineTrainStep, ResNet50Engine

N = int(sys.argv[1]) if len(sys.argv) > 1 else 256
inline = len(sys.argv) > 2 and sys.argv[2] == "inline"   # weight-gradient GEMMs in line: clean per-kernel durations
eng = ResNet50Engine(batch=N, num_classes=1000, overlap_wgrad=not inline)
step = EngineTrainStep(eng, optim.SGD(0.1, momentum=0.9), use_graph=False)
x = torch.randint(0, 256, (N, 224, 224, 3), device="cuda", dtype=torch.uint8)
y = torch.randint(0, 1000, (N,), device="cuda")
step.load(x, y)
for _ in range(3):
    step.run()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(3):
        step.run()
    torch.cuda.synchronize()
tab = prof.key_averages().table(sort_by="cuda_time_total", row_limit=45, max_name_column_width=90)
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles")
os.makedirs(OUT, exist_ok=True)
with open(os.path.join(OUT, "step_profile.txt"), "w") as f:
    f.write(tab)
# compact per-kernel summary (3 steps)
rows = [(e.key, e.device_time_total / 3.0, e.count // 3) for e in prof.key_averages() if e.device_time_total > 0 and e.device_type.name == "CUDA"]
rows.sort(key=lambda r: -r[1])
tot = sum(r[1] for r in rows)
with open(os.path.join(OUT, "step_kernels.txt"), "w") as f:
    f.write(f"total device kernel time per step: {tot/1e3:.2f} ms\n")
    for k, t, c in rows[:60]:
        f.write(f"{t/1e3:9.3f} ms  {100*t/tot:5.1f}%  x{c:<4d} {k[:150]}\n")
print(open(os.path.join(OUT, "step_kernels.txt")).read())
