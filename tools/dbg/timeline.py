"""Per-warp timeline of the cooperative HP1 step (debug build: python tools/build_variant.py timeline --hp1 "-DAGX_TIMELINE"):
    AGX_LIB_PATH=tools/dbg/libagx_timeline.so python tools/dbg/timeline.py"""
import ctypes as C
import sys
import numpy as np
import torch
sys.path.insert(0, ".")
from aerial_gym_simulator_b200 import _lib
from aerial_gym_simulator_b200.hp1 import Hp1Engine, MultirotorSpec

dev = torch.device("cuda:0")
N = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
spec = MultirotorSpec()
R = 16
engs = []
for r in range(R):
    e = Hp1Engine(spec, N, dev, seed=1 + r, materialize_derived=False)
    e.reset(torch.ones(N, dtype=torch.bool, device=dev))
    e.refresh()
    e.sim_steps.copy_((torch.arange(N, device=dev) % 500).int())
    engs.append(e)
acts = [torch.rand(N, 4, device=dev) * 2 - 1 for _ in range(8)]
lib = _lib.load()
lib.agx_dbg_timeline.argtypes = [C.c_void_p]
for i in range(64):
    engs[i % R].position_task_step(acts[i % 8])
torch.cuda.synchronize()
out = np.zeros((7, 8192), dtype=np.uint64)  # g_timeline[7][8192] (hp1.cu)
W = (N + 31) // 32
rows = []
NREP = int(sys.argv[2]) if len(sys.argv) > 2 else 5
BRIEF = NREP > 5
for rep in range(NREP):
    e = engs[rep % R]
    n_trunc_pred = int((e.sim_steps >= 500).sum())
    ar0 = e.any_reset.cpu().tolist()
    e.position_task_step(acts[rep % 8])
    torch.cuda.synchronize()
    _lib.check(lib.agx_dbg_timeline(out.ctypes.data_as(C.c_void_p)))
    t = out[:, :W].astype(np.int64)
    t0 = t[0].min()
    t = (t - t0) / 1e3
    reset = e.reset_mask.view(-1, 32).any(1).cpu().numpy() if N % 32 == 0 else None
    q = lambda a: " ".join(f"{np.percentile(a, p):6.2f}" for p in (0, 10, 50, 90, 99, 100))
    if BRIEF:
        ar1 = e.any_reset.cpu().tolist()
        print(f"rep {rep:2d} eng {rep % R:2d}: span {t[3].max():6.2f}  physics p50 {np.median(t[1]-t[0]):5.2f}  epi p50 {np.median(t[2]-t[1]):5.2f} "
              f"end p50 {np.median(t[3]):6.2f}  pred_trunc {n_trunc_pred}  resets {int(e.reset_mask.sum())} crashes {int(e.terminations.sum())} "
              f"any_reset before {ar0[2:6]} after {ar1[2:6]}")
        continue
    print(f"rep {rep}: kernel span {t[3].max():.2f} us; percentiles 0/10/50/90/99/100")
    print("   warp start      :", q(t[0]))
    print("   physics done    :", q(t[1]))
    print("   epilogue done   :", q(t[2]))
    print("   warp end        :", q(t[3]))
    print("   warp duration   :", q(t[3] - t[0]), " physics:", q(t[1] - t[0]), " epilogue:", q(t[2] - t[1]), " tail:", q(t[3] - t[2]))
    if reset is not None:
        print(f"   warps with a reset: {reset.sum()}  their epilogue:", q((t[2] - t[1])[reset]), " end:", q(t[3][reset]))
        print("   warps without      their end:", q(t[3][~reset]))
