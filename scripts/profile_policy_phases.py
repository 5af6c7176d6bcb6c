"""Per-phase clock64 breakdown of the fused policy kernel (thread 0 of every CTA): python scripts/profile_policy_phases.py [R]"""
import sys

import torch

sys.path.insert(0, ".")
from deeprl_signal_control_b200 import _lib
from deeprl_signal_control_b200.agents.layout import PolicyLayout
from deeprl_signal_control_b200.agents.learner import BatchedA2C
from deeprl_signal_control_b200.net.large_grid import build_large_grid

R = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
net = build_large_grid(agent="ma2c")
lay = PolicyLayout(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, net.node_obs_off, net.n_obs, fw=128, ft=32, ff=64, h=64)
# consumer 0 (items of even parity) and the producer warpgroup, thread 0 of each
names = ["consumer: unit constants", "consumer: wait for staged operands", "consumer: MMA0 + wait",
         "consumer: relu epilogue, h staging, st_x", "consumer: gate MMA + wait", "consumer: cell, stores, heads"]
pnames = ["producer: unit constants", "producer: wait for a free tile", "producer: fc copy + obs staging"]
for store in (True, False):
    m = BatchedA2C(lay, R, n_step=8, seed=1, store_acts=store)
    obs = torch.rand(R, lay.n_obs, device="cuda")
    for _ in range(3):
        m.t = 0
        m.forward(obs, False)
    prof = torch.zeros(16, dtype=torch.int64, device="cuda")
    lib = _lib.lib()
    lib.tscl_debug_policy_prof(prof.data_ptr())
    n = 4
    for i in range(n):
        m.t = i
        m.forward(obs, False)
    torch.cuda.synchronize()
    lib.tscl_debug_policy_prof(None)
    n_cta = min(((R + 63) // 64) * 2 * lay.A, torch.cuda.get_device_properties(0).multi_processor_count)
    pa = prof.cpu().numpy().astype(float) / n / n_cta
    for who, nm_list, p in (("consumer 0", names, pa[:6]), ("producer", pnames, pa[8:11])):
        tot = p.sum()
        print("activation store %s, %s: %.0f cycles per CTA per launch" % (store, who, tot))
        for nm, v in zip(nm_list, p):
            print("   %-42s %9.0f cycles  %5.1f %%" % (nm, v, 100 * v / tot))
    del m
