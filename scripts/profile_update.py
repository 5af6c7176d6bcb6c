"""Per-kernel breakdown of one A2C update of the bench workload (5x5 grid MA2C, R = 4096, update chunks of 1024 replicas,
n_step 120, seed 12 as in bench.py), measured with torch.profiler (CUDA activities):

    python scripts/profile_update.py          # trace under $OUT (default results/)

One line per kernel name: total ms inside the update, launches, and achieved GB/s where the script knows the bytes the
kernel has to move (computed below from the shapes).  The card, its power limit and the SM clock are read in the same run.
"""
import json
import os
import subprocess
import sys
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler, make_layout  # noqa: E402
from deeprl_signal_control_b200.agents.learner import BatchedA2C  # noqa: E402
from deeprl_signal_control_b200.agents.trainer import BatchedTrainer  # noqa: E402
from deeprl_signal_control_b200.net.large_grid import build_large_grid  # noqa: E402
from deeprl_signal_control_b200.net.tables import EnvParams  # noqa: E402
from deeprl_signal_control_b200.sim import BatchedSim  # noqa: E402

R, CHUNK, T, SEED = 4096, 1024, 120, 12
OUT = os.environ.get("OUT", "results")
os.makedirs(OUT, exist_ok=True)


class _Args:
    agent, policy = "ma2c", "lstm"


net, par = build_large_grid(agent="ma2c"), EnvParams(agent="ma2c")
lay = make_layout(net, _Args)
sim = BatchedSim(net, par, R, device=0)
m = BatchedA2C(lay, R, n_step=T, gamma=0.99, v_coef=0.5, max_grad_norm=40.0, alpha=0.99, eps=1e-5, reward_norm=2000.0,
               reward_clip=2.0, seed=SEED, device=0, chunk=CHUNK)
tr = BatchedTrainer(sim, m, "ma2c", lr=5e-4, beta=0.01, seed0=SEED)

# essential HBM bytes per update chunk (U units, M = T * rc rows): each operand read once, each result written once
U, dx, H = 2 * lay.A, lay.dx, lay.h
M = T * CHUNK
n_chunks = (R + CHUNK - 1) // CHUNK
BYTES = {   # per update
    "wgrad_tc_async_kernel": n_chunks * U * M * (4 * H * 2 + dx * 2 + H * 2),     # dZ, X, Hp (bf16)
    "dx_tc_kernel": n_chunks * U * M * (4 * H * 2 + dx * 2),                      # dZ in, dX out (bf16)
    "fc_bwd_tc_kernel": n_chunks * U * M * (dx * 2 + dx * 2),                     # dX, X (bf16)
    # dZ, X (bf16); the observation slice (fp32, shared by an agent's two units and read through L2) is not counted
    "dx_fc_bwd_tc_kernel": n_chunks * U * M * (4 * H * 2 + dx * 2),
    # gates, c, then h_t (bf16) when the kernel computes dH itself (heads_in_bptt) or dH (fp32) in; dZ out
    "lstm_bwd_tc_regs_kernel": n_chunks * U * M * (4 * H * 2 + H * 2 + (H * 2 if m.heads_in_bptt else H * 4) + 4 * H * 2),
    "heads_loss_kernel": n_chunks * U * M * (H * 2 + H * 4),                      # h (bf16) in, dH (fp32) out
}
print("heads in the BPTT kernel: %s (TSC_BPTT_HEADS=0 runs heads_loss_kernel + the BPTT per chunk)" % m.heads_in_bptt)

assert m.store_acts, "the bf16 activation store does not fit: the update would take the fp32 path"
tr.run(T)                              # one rollout + one update: warms up every shape of the update
tr.update_events = []
tr.run(T)                              # one more, timed with CUDA events only
torch.cuda.synchronize()
upd_ms_events = tr.update_events[0][0].elapsed_time(tr.update_events[0][1])
tr.update_events = None
tr.run(T - 1)
torch.cuda.synchronize()
assert all(m._acts_ok[:T - 1]), "the rollout did not fill the bf16 activation store"
sampler = ClockSampler(0)
sampler.start()
prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
update = tr.update


def profiled_update():                 # the profiler sees the update's kernels and nothing else
    torch.cuda.synchronize()
    prof.start()
    update()
    torch.cuda.synchronize()
    prof.stop()


tr.update = profiled_update
tr.run(1)                              # the T-th control step, then the update
tr.update = update
sampler.stop_flag = True
sampler.join(timeout=2)
trace = os.path.join(OUT, "update_trace.json")
prof.export_chrome_trace(trace)

agg = defaultdict(lambda: [0.0, 0])
for ev in json.load(open(trace))["traceEvents"]:
    if ev.get("cat") == "kernel":
        name = ev["name"].split("(")[0].split("<")[0].replace("void ", "")
        agg[name][0] += ev["dur"] * 1e-3
        agg[name][1] += 1
tot = sum(v[0] for v in agg.values())

smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
clk = sampler.summary()
print("card: %s | SM clock during the profiled update: %s MHz (max %s)%s" %
      (smi, clk["sm_mhz"], clk["sm_max_mhz"], (", " + ",".join(clk["reasons"])) if clk["reasons"] else ""))
print("update: %.2f ms (CUDA events, unprofiled); kernel time in the profiled update: %.2f ms" % (upd_ms_events, tot))
print("%-34s %9s %7s %6s %9s" % ("kernel", "ms", "launches", "%", "GB/s"))
for name, (ms, n) in sorted(agg.items(), key=lambda x: -x[1][0]):
    gbs = "%9.0f" % (BYTES[name] / (ms * 1e-3) / 1e9) if name in BYTES else "        -"
    print("%-34s %9.2f %7d %6.1f %s" % (name[:34], ms, n, 100 * ms / tot, gbs))
three = sum(agg[k][0] for k in ("wgrad_tc_async_kernel", "dx_tc_kernel", "fc_bwd_tc_kernel", "dx_fc_bwd_tc_kernel")
            if k in agg)
print("wgrad + dx + fc_bwd (or dx_fc_bwd): %.2f ms = %.1f %% of the update's kernel time" % (three, 100 * three / tot))
