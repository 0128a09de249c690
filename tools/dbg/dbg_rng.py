import os
import torch, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import aerial_gym_simulator_b200.task
from aerial_gym_simulator_b200.registry.task_registry import task_registry
cfg = task_registry.get_task_config("position_setpoint_task")
cfg.args = {"reset_rng": "torch"}
task = task_registry.make_task("position_setpoint_task", seed=5, num_envs=64, headless=True)
torch.manual_seed(1234)
import torch as T
orig = T.rand
outs=[]
def spy(*a, **k):
    out = orig(*a, **k); outs.append(out.clone()); return out
T.rand = spy
task.reset()
T.rand = orig
torch.cuda.synchronize()
eng=task.sim_env.engine
print("state row0", eng.root_state[0])
print("spy state draw row0", outs[2][0])
torch.manual_seed(1234)
a=torch.rand(64,3,device="cuda:0"); b=torch.rand(64,3,device="cuda:0"); c=torch.rand(64,13,device="cuda:0")
print("replay row0", c[0])
print("a equal", torch.equal(a, outs[0]), torch.equal(b, outs[1]), torch.equal(c, outs[2]))
lo=torch.tensor(task.sim_env.spec.min_init_state,device="cuda:0"); hi=torch.tensor(task.sim_env.spec.max_init_state,device="cuda:0")
rs=(hi-lo)*outs[2]+lo
print("expected pos from spy", (-1+2*rs[0,0:3]))
