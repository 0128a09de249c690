import os
import sys, time, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from aerial_gym_simulator_b200.hp1 import Hp1Engine, MultirotorSpec
dev = torch.device("cuda:0")
N = 65536
eng = Hp1Engine(MultirotorSpec(), N, dev, seed=1, materialize_derived=False)
eng.reset(torch.ones(N, dtype=torch.bool, device=dev)); eng.refresh()
eng.sim_steps.copy_((torch.arange(N, device=dev) % 500).int())
a = (torch.rand(N, 4, device=dev) * 2 - 1).contiguous()
for _ in range(50): eng.position_task_step(a)
torch.cuda.synchronize()
K = 2000
t0 = time.perf_counter()
for _ in range(K): eng.position_task_step(a)
t_cpu = time.perf_counter() - t0
torch.cuda.synchronize()
t_all = time.perf_counter() - t0
print(f"eager: cpu issue {t_cpu/K*1e6:.1f} us/step, incl gpu drain {t_all/K*1e6:.1f} us/step")
# graph
g = torch.cuda.CUDAGraph()
s = torch.cuda.Stream()
s.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(s):
    for _ in range(3): eng.position_task_step(a)
torch.cuda.current_stream().wait_stream(s)
with torch.cuda.graph(g, stream=s):
    eng.position_task_step(a)
torch.cuda.synchronize()
for _ in range(50): g.replay()
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(K): g.replay()
t_cpu = time.perf_counter() - t0
torch.cuda.synchronize()
t_all = time.perf_counter() - t0
print(f"graph: cpu issue {t_cpu/K*1e6:.1f} us/step, incl gpu drain {t_all/K*1e6:.1f} us/step")
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(K): g.replay()
e1.record(); torch.cuda.synchronize()
print(f"graph: gpu events {e0.elapsed_time(e1)/K*1e3:.2f} us/step")
