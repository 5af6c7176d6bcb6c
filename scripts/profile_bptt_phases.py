"""Per-phase clock64 breakdown of the store-path BPTT kernel (lstm_bwd_tc_regs_kernel: thread 0 of every warpgroup) during
one update: python scripts/profile_bptt_phases.py [R] [chunk]"""
import sys

import torch

sys.path.insert(0, ".")
from deeprl_signal_control_b200 import _lib
from deeprl_signal_control_b200.agents.layout import PolicyLayout
from deeprl_signal_control_b200.agents.learner import BatchedA2C
from deeprl_signal_control_b200.agents.trainer import BatchedTrainer
from deeprl_signal_control_b200.net.large_grid import build_large_grid
from deeprl_signal_control_b200.net.tables import EnvParams
from deeprl_signal_control_b200.sim import BatchedSim

R = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
chunk = int(sys.argv[2]) if len(sys.argv) > 2 else 4096
net, par = build_large_grid(agent="ma2c"), EnvParams(agent="ma2c")
lay = PolicyLayout(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, net.node_obs_off, net.n_obs, fw=128, ft=32, ff=64, h=64)
sim = BatchedSim(net, par, R)
m = BatchedA2C(lay, R, n_step=120, reward_norm=2000.0, reward_clip=2.0, seed=1, chunk=chunk)
tr = BatchedTrainer(sim, m, "ma2c", lr=5e-4, beta=0.01, seed0=12)
tr.run(120)                       # one rollout + one update (warm-up)
tr.run(119)
torch.cuda.synchronize()
prof = torch.zeros(8, dtype=torch.int64, device="cuda")
_lib.lib().tscl_debug_bptt_prof(prof.data_ptr())
tr.run(1)                         # the 120th step triggers the update
torch.cuda.synchronize()
_lib.lib().tscl_debug_bptt_prof(None)
n_sm = torch.cuda.get_device_properties(0).multi_processor_count
n_items = 2 * lay.A * ((chunk + 127) // 128) * ((R + chunk - 1) // chunk)
n_cta = min(n_items, n_sm)                      # persistent grid, two warpgroups per CTA
wg_steps = 2 * lay.A * ((R + chunk - 1) // chunk) * ((chunk + 63) // 64) * 120   # (64-row slab, step) pairs
p = prof.cpu().numpy()[:4].astype(float) / (2 * n_cta)
tot = p.sum()
steps = wg_steps / (2 * n_cta)
print("BPTT: %.0f cycles per warpgroup per update, %.0f (64-row slab, step) pairs per warpgroup = %.0f cycles each"
      % (tot, steps, tot / steps))
for nm, v in zip(["wait for step t's operands", "smem -> regs, operand issue, cell backward",
                  "MMA issue -> wait", "dZ store (stmatrix, barrier, TMA store issue)"], p):
    print("   %-48s %9.0f cycles  %5.1f %%   %.0f per step" % (nm, v, 100 * v / tot, v / steps))
