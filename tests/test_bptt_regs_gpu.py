"""GPU: the store-path BPTT kernel that keeps the recurrence in registers (lstm_bwd_tc_regs_kernel, the default of
tscl_lstm_seq_bwd_tc with gates / c / dZ in bf16) gives the dZb of lstm_bwd_tc_kernel<512> (TSC_BPTT_STAGED=0) bit
for bit, and writes nothing past the last row of dZb.

Both kernels use the same operands, k-step order, per-element formulas and bf16 rounding points, so any difference is a
defect, not rounding.  The kernel-selection switch is read once per process, so each kernel runs in a fresh subprocess
that writes the sha256 of dZb per done pattern."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GUARD = 4096                    # bf16 elements allocated after dZb's last row
SENTINEL = 0x7FC1               # a bf16 NaN the kernels never produce


def _digests(out_path, kind, T, Rc, ld, r0):
    """dZb digests for done patterns {37, 90}, {0, T-1} and all-done, whether the guard after dZb is intact, and whether
    the register-recurrence kernel is the one that ran (it adds to the phase counters, lstm_bwd_tc_kernel does not)."""
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import _p
    from tests.test_update_bench_size_gpu import _bptt_inputs, _model
    lay, m = _model(kind)
    U = lay.U
    n = U * T * Rc * 256
    res = {"digests": [], "guard_ok": True, "all_written": True}
    for pat, steps in enumerate([(37 % T, 90 % T), (0, T - 1), tuple(range(T))]):
        gates, cb, dH, c_bw, done = _bptt_inputs(U, T, Rc, ld, steps, seed=20 + pat)
        buf = torch.empty(n + GUARD, dtype=torch.bfloat16, device="cuda")
        buf.view(torch.int16).fill_(SENTINEL)
        dZb = buf[:n].view(U, T * Rc, 256)
        _lib.check(_lib.lib().tscl_lstm_seq_bwd_tc(
            m._h, _p(m.Wt), None, None, _p(dH), _p(c_bw), _p(done), C.c_int32(T), C.c_int64(Rc), C.c_int64(ld),
            C.c_int64(r0), _p(gates), _p(cb), _p(dZb), m._st()))
        torch.cuda.synchronize()
        res["digests"].append(hashlib.sha256(dZb.view(torch.int16).cpu().numpy().tobytes()).hexdigest())
        res["guard_ok"] &= bool((buf[n:].view(torch.int16) == SENTINEL).all())
        res["all_written"] &= not bool((dZb.view(torch.int16) == SENTINEL).any())
        del gates, cb, dH, c_bw, done, buf, dZb
    prof = torch.zeros(8, dtype=torch.int64, device="cuda")
    gates, cb, dH, c_bw, done = _bptt_inputs(U, 2, 64, 64, (), seed=1)
    dZb = torch.empty(U, 2 * 64, 256, dtype=torch.bfloat16, device="cuda")
    _lib.lib().tscl_debug_bptt_prof(C.c_void_p(prof.data_ptr()))
    _lib.check(_lib.lib().tscl_lstm_seq_bwd_tc(
        m._h, _p(m.Wt), None, None, _p(dH), _p(c_bw), _p(done), C.c_int32(2), C.c_int64(64), C.c_int64(64),
        C.c_int64(0), _p(gates), _p(cb), _p(dZb), m._st()))
    torch.cuda.synchronize()
    _lib.lib().tscl_debug_bptt_prof(None)
    res["regs_kernel_ran"] = bool(prof.sum().item() > 0)
    with open(out_path, "w") as f:
        json.dump(res, f)


def _run(tmp_path, env, args):
    out = tmp_path / ("%s%s.json" % ("_".join(str(a) for a in args), "_ref" if env else ""))
    e = {k: v for k, v in os.environ.items() if not k.startswith("TSC_BPTT_")}
    e.update(env)
    r = subprocess.run([sys.executable, "-c", "import sys, json; from tests.test_bptt_regs_gpu import _digests; "
                        "_digests(sys.argv[1], sys.argv[2], *map(int, sys.argv[3:]))", str(out)] + [str(a) for a in args],
                       cwd=ROOT, env=e, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(out.read_text())


@pytest.mark.parametrize("kind,T,Rc,ld,r0", [
    ("grid", 120, 1024, 2048, 1024),     # the bench chunk
    ("monaco", 40, 1024, 2048, 1024),
    ("grid", 120, 1000, 3000, 1000),     # ragged last tile (104 rows: the second warpgroup has 40)
    ("grid", 120, 100, 200, 100),        # one partial tile: the second warpgroup has 36 rows
    ("grid", 120, 40, 80, 40),           # one partial tile: the second warpgroup has no row
])
def test_regs_kernel_bit_identical_to_reference_kernel(tmp_path, kind, T, Rc, ld, r0):
    new = _run(tmp_path, {}, (kind, T, Rc, ld, r0))
    ref = _run(tmp_path, {"TSC_BPTT_STAGED": "0"}, (kind, T, Rc, ld, r0))
    assert new["regs_kernel_ran"] and not ref["regs_kernel_ran"]
    assert new["guard_ok"] and ref["guard_ok"]
    assert new["all_written"] and ref["all_written"]
    for pat, (a, b) in enumerate(zip(new["digests"], ref["digests"])):
        assert a == b, "done pattern %d: dZb differs" % pat
