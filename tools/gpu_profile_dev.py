"""Dev script (GPU box): in-kernel phase profile of one batch solve of the bench workload (configs[1]: hill, 1024 problems), and the
slot efficiency of its solve launches.

Slot efficiency = (summed per-problem PF_TOTAL cycles) / (resident trajectory slots x elapsed cycles): the share of the slot time
the device holds that trajectories spend being solved.  Elapsed cycles are the solve's event time times the SM clock that
nvidia-smi reports while the solve runs.  Resident slots assume the bench's launch plan: every trajectory in a two-warp group,
two slots per CTA, two CTAs per SM."""
import os, subprocess, sys
import ctypes as C
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from uneven_planner_b200 import maps, problems, _lib, api, configs
import torch

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
m = maps.get_terrain("hill", build_if_missing=False) or maps.synthetic_terrain("bumps", seed=0)
pb = problems.generate(m, B, seed=0, **configs.gen_kwargs("hill"))
opt = api.BatchALMTrajOpt().init(configs.params_for("hill")).set_environment(m)
opt.upload(pb)
opt.profile(True)
clock_mhz = []
for rep in range(3):
    opt.solve_resident()
    clock_mhz.append(float(subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                                          capture_output=True, text=True).stdout.split()[0]))
    opt.sync()
ms, _ = opt.last_solve_ms()
raw = (C.c_longlong * (16 * B))()
api._check(opt.L.ualm_profile(opt.h, 2, raw))
per = np.frombuffer(raw, dtype=np.int64).reshape(B, 16)
pr = opt.profile(True, read=True)
res, _, _ = opt.download()
ev = sum(r.n_evals for r in res); it = sum(r.n_lbfgs_iters for r in res)
tot = pr["total"]
print(f"B={B} kernel {ms:.1f} ms; evals {ev} iters {it}; mean cycles/traj {tot/B:.3e}; cycles/eval {tot/ev:.0f}")
for k, v in pr.items():
    print(f"  {k:12s} {100.0*v/tot:6.2f}%   {v/ev:10.0f} cyc/eval")
sms = torch.cuda.get_device_properties(0).multi_processor_count
slots = min(B, 2 * 2 * sms)
mhz = float(np.median(clock_mhz))
busy = float(per[:, 15].sum())
print(f"slot efficiency {busy / (slots * ms * 1e3 * mhz):.3f}: {busy:.4e} trajectory cycles over {slots} slots x {ms:.1f} ms at {mhz:.0f} MHz "
      f"(SM clock samples {clock_mhz}); per-trajectory cycles p50 {np.median(per[:, 15]):.3e} max {per[:, 15].max():.3e}")
