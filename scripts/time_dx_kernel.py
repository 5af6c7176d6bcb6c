"""Times tscl_dx_tc against the library product on one update chunk (grid MA2C: 50 units x 122 880 rows): python scripts/time_dx_kernel.py"""
import sys

import torch

sys.path.insert(0, ".")
from deeprl_signal_control_b200 import _lib
from deeprl_signal_control_b200.agents.layout import PolicyLayout
from deeprl_signal_control_b200.agents.learner import BatchedA2C
from deeprl_signal_control_b200.net.large_grid import build_large_grid

net = build_large_grid(agent="ma2c")
lay = PolicyLayout(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, net.node_obs_off, net.n_obs, fw=128, ft=32, ff=64, h=64)
m = BatchedA2C(lay, 128, n_step=2, seed=1)
U, dx, M = lay.U, lay.dx, 1024 * 120
dZ = (torch.randn(U, M, 256, device="cuda") * 0.1).to(torch.bfloat16)
dX = torch.empty(U, M, dx, device="cuda", dtype=torch.bfloat16)
wxb = m.pv["wx"].to(torch.bfloat16)
st = _lib.stream()
own = lambda: _lib.check(_lib.lib().tscl_dx_tc(m._h, dZ.data_ptr(), m.Wxt.data_ptr(), dX.data_ptr(), M, st))
libf = lambda: torch.bmm(dZ, wxb.transpose(1, 2), out=dX)
nbytes = U * M * (256 + dx) * 2
for name, f in (("tscl_dx_tc", own), ("torch.bmm", libf)):
    for _ in range(3):
        f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        f()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print("%-12s %.3f ms per chunk  %.0f GB/s" % (name, ms, nbytes / ms / 1e6))
