"""Time the fused policy forward (tscl_policy_step_v2) alone at the bench shapes, with CUDA events:

    python scripts/profile_policy_forward.py [--launches N]

Three cases: the rollout forward of the 5x5 grid MA2C (R = 4096, bf16 activation store on), the bootstrap forward of the
same model (out_type 'v': no store, no sample, state written to the scratch buffers) and Monaco MA2C (R = 2048, store
on).  For each: ms per launch over N launches after a warm-up, the HBM bytes the kernel has to move (computed below
from the shapes: every operand read once, every result written once), the achieved GB/s and its share of the H100 SXM
data-sheet 3.35 TB/s.  The card and its power limit are read in the same run.
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import build_scenario, make_layout  # noqa: E402
from deeprl_signal_control_b200.agents.learner import BatchedA2C  # noqa: E402

HBM_PEAK = 3.35e12


def forward_bytes(lay, R, store, out_type):
    """Essential HBM traffic of one launch, by array (bytes)."""
    U, H = lay.U, lay.h
    b = {"obs": R * lay.n_obs * 4,
         "c_in, h_in (fp32)": 2 * U * R * H * 4,
         "c_out, h_out (fp32)": 2 * U * R * H * 4}
    if store:
        b["st_x"] = U * R * lay.dx * 2
        b["st_g"] = U * R * 4 * H * 2
        b["st_c + st_h"] = 2 * U * R * H * 2
    b["pi, val, act"] = R * lay.A * (lay.max_na * 4 + 4 + (4 if "p" in out_type else 0))
    return b


def time_case(name, scenario, R, out_type, launches, warmup):
    class _Args:
        agent, policy = "ma2c", "lstm"
    _Args.scenario = scenario
    net = build_scenario(_Args)[0]
    lay = make_layout(net, _Args)
    store = "p" in out_type
    m = BatchedA2C(lay, R, n_step=2, seed=1, chunk=1024, store_acts=store)
    assert m.tc_v2 and m.store_acts == store
    g = torch.Generator(device="cuda").manual_seed(0)
    obs = torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2
    m.t = 1                                     # store slot 1 of 2: chunk index >= 1 for R > 1024

    def run(n):
        for _ in range(n):
            m.forward(obs, False, out_type=out_type)

    run(warmup)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run(launches)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / launches
    b = forward_bytes(lay, R, store, out_type)
    tot = sum(b.values())
    gbs = tot / (ms * 1e-3) / 1e9
    print("%s: R = %d, %d units, dx = %d: %.4f ms per launch (%d launches), %.0f MB, %.0f GB/s = %.1f %% of 3.35 TB/s"
          % (name, R, lay.U, lay.dx, ms, launches, tot / 1e6, gbs, 100 * gbs * 1e9 / HBM_PEAK))
    for k, v in b.items():
        print("    %-22s %8.1f MB" % (k, v / 1e6))
    del m
    return ms


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--launches", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    args = p.parse_args()
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("card: %s | library: %s" % (smi, os.environ.get("TSC_LIB", "in-tree libtsc.so")))
    time_case("grid MA2C rollout (store on)", "large_grid", 4096, "pv", args.launches, args.warmup)
    time_case("grid MA2C bootstrap (out_type 'v')", "large_grid", 4096, "v", args.launches, args.warmup)
    time_case("Monaco MA2C rollout (store on)", "real_net", 2048, "pv", args.launches, args.warmup)


if __name__ == "__main__":
    main()
