"""Unit-queue mode (b2s_set_mode 2) on Lift: the small role's stage counters (mean clock64 cycles per block round and share of each
stage), the ring counters of the last control step and the warn bits.  Needs the -DB2S_INSTR build of the library, which registers
the arrays "unit_prof" and "unit_ctr": B2S_LIB=robosuite_b200/variants/libb2s_instr.so (robosuite_b200.build.build_instr()).
usage: python tools/probe_unit.py [n_env] [control steps]"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import robosuite_b200 as suite  # noqa: E402

STAGES = ["take tickets", "ring slots", "phase 0", "narrow phase", "rows (gather, constraint)", "controller",
          "actuation + acceleration", "solve", "integrate, obs, publish"]
NSUB = 25

if "B2S_LIB" not in os.environ:
    sys.exit("probe_unit.py needs the -DB2S_INSTR library: B2S_LIB=robosuite_b200/variants/libb2s_instr.so")
n = int(sys.argv[1]) if len(sys.argv) > 1 else 16
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
env = suite.make("Lift", robots="Panda", num_envs=n, seed=1, horizon=10 ** 9)
sim = env.sim
sim.set_mode(2)
gen = torch.Generator(device=env.device)
gen.manual_seed(3)
for i in range(steps):
    sim.env_step(torch.rand((n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1, NSUB)
torch.cuda.synchronize()
h = sim.unit_prof.cpu().tolist()
rounds, tot = h[15], max(sum(h[:9]), 1)
print("unit-queue stage profile over %d block rounds (mean cycles per round, share):" % rounds)
for k, nm in enumerate(STAGES):
    print("  %-28s %9.0f  %5.1f %%" % (nm, h[k] / max(rounds, 1), 100.0 * h[k] / tot))
c = sim.unit_ctr.cpu().tolist()
print("ring counters of the last control step: head %d tail %d done %d ovf_head %d ovf_tail %d | watchdog ticket %d tail_then %d "
      "flag %d (total %d)" % (*c, n * NSUB))
print("warn", int(sim.warn.abs().max()))
