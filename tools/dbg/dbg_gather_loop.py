"""1-GPU loopback timing of the chained steps with / without the observation gather attached (emulated world: pushes go to local buffers)."""
import os
import sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from aerial_gym_simulator_b200.distributed import PipelinedObsGather
from aerial_gym_simulator_b200.hp1 import Hp1Engine, MultirotorSpec
from aerial_gym_simulator_b200 import _lib
DEV='cuda:0'; n=65536
_lib.check(_lib.load().agx_set_spin_timeout_ms(3000), "t")
def run(R, lb, ctas=24, nb=4, steps=200):
    engines = []
    for r in range(R):
        e = Hp1Engine(MultirotorSpec(), n, DEV, seed=9 + r, materialize_derived=False)
        e.reset(torch.ones(n, dtype=torch.bool, device=DEV)); e.refresh()
        e.sim_steps.copy_((torch.arange(n, device=DEV) % 500).int())
        engines.append(e)
    gth = None
    if lb:
        gth = PipelinedObsGather(n, 13, DEV, num_buffers=nb, loopback_world=lb, max_ctas=ctas)
        for e in engines: e.attach_obs_gather(gth)
    act = torch.zeros(n, 4, device=DEV)
    def loop(k):
        for i in range(k): engines[i % R].position_task_step(act)
        if gth is not None:
            gth.loopback_complete(gth.epoch); gth.fence(); gth.wait()
    loop(32); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    import time; t0 = time.perf_counter()
    e0.record(); loop(steps); e1.record(); th = time.perf_counter() - t0
    torch.cuda.synchronize()
    err = hex(gth.error_word.item()) if gth is not None else None
    engerr = [hex(e.any_reset[2].item()) for e in engines if e.any_reset[2].item()]
    print(f"replicas={R} loopback_world={lb} ctas={ctas} ring={nb}: {e0.elapsed_time(e1) * 1e3 / steps:.2f} us/step, host enqueue {th * 1e6 / steps:.2f} us/step, gather err {err}, engine errs {engerr}", flush=True)
import os
if os.environ.get("ONLY") == "ncu":
    _lib.check(_lib.load().agx_set_spin_timeout_ms(120000), "t")
    run(16, 2, steps=60)
else:
    run(1, 0); run(16, 0); run(1, 2); run(16, 2); run(16, 4); run(16, 8); run(16, 2, ctas=8); run(16, 2, ctas=48, nb=2)
