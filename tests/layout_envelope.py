"""Layouts of tests/test_layout_envelope_cpu.py and tests/test_layout_envelope_gpu.py: the shipped scenarios at the
reference's model widths (num_fw 128, num_ft 32, num_fp 64, num_lstm 64), built the way agents/models.py IA2C / MA2C
build them, and synthetic layouts at the edges of what the tensor-core kernels accept (tscl_create: wave blocks of at
most 48 inputs, 16 fingerprint and 16 wait inputs, 8 actions; the 64-slot input tile of the fused kernels).

Each entry names the forward family and update path learner_paths selects for it (agents/learner.py)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FW, FT, FP, LSTM = 128, 32, 64, 64


def net_tables(scenario, agent, mini_dir=None):
    if scenario == "large_grid":
        from deeprl_signal_control_b200.net.large_grid import build_large_grid
        return build_large_grid(agent=agent)
    if scenario == "real_net":
        from deeprl_signal_control_b200.net.real_net import real_net_tables
        return real_net_tables(agent)
    if scenario == "small_grid":
        from deeprl_signal_control_b200.net.small_grid import build_small_grid
        return build_small_grid(agent=agent)
    assert scenario == "mini_sumo", scenario
    sys.path.insert(0, os.path.join(ROOT, "tests", "fixtures"))
    import make_mini_sumo
    from deeprl_signal_control_b200.net import sumo_ingest
    return sumo_ingest.load_sumo_scenario(*make_mini_sumo.write(mini_dir), agent=agent, use_wait=True)


def scenario_layout(net, agent, fw=FW):
    """models.IA2C / MA2C: the fingerprint block for MA2C only, max_na from the agents' action counts"""
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    return PolicyLayout(net.n_s_ls, net.n_a_ls, net.n_w_ls, net.n_f_ls, net.node_obs_off, net.n_obs, fw=fw, ft=FT,
                        ff=FP if agent == "ma2c" else 0, h=LSTM)


def synthetic_layout(n_wave, n_wait, n_fp, n_a, fw=FW, ft=FT, ff=0, max_na=None):
    """agents with the given input blocks, observation vectors back to back (wave | wait | fingerprint) plus 3 spare
    floats at the end"""
    from deeprl_signal_control_b200.agents.layout import PolicyLayout
    n_s = [w + t + f for w, t, f in zip(n_wave, n_wait, n_fp)]
    off = np.concatenate([[0], np.cumsum(n_s)]).astype(np.int32)
    return PolicyLayout(n_s, n_a, n_wait, n_fp, off, int(off[-1]) + 3, fw=fw, ft=ft, ff=ff, h=LSTM, max_na=max_na)


# scenario, agent, fw -> (forward, update with the activation store on)
SCENARIOS = {
    ("large_grid", "ma2c", FW): ("v2", "lean"),            # dx 224
    ("large_grid", "ia2c", FW): ("v2", "lean"),            # dx 160
    ("large_grid", "ia2c", 96): ("v2", "lean"),            # dx 128
    ("large_grid", "ia2c", 64): ("v1", "recompute"),       # dx 96: outside the v2 widths, wave block <= 32
    ("real_net", "ma2c", FW): ("v2", "lean"),              # dx 192, wave block 48
    ("real_net", "ia2c", FW): ("v2", "lean"),              # dx 128 (no wait, no fingerprint block), wave block 48
    ("small_grid", "ma2c", FW): ("v2", "lean"),
    ("small_grid", "ia2c", FW): ("v2", "lean"),
    ("mini_sumo", "ma2c", FW): ("v2", "lean"),
    ("mini_sumo", "ia2c", FW): ("v2", "lean"),
}

# synthetic edges: name -> (layout kwargs, forward, update)
EDGES = {
    # widest wave block 32 with wait inputs: the block fills the 32-wide tile, no spare slot for the bias column
    "wave32_wait": (dict(n_wave=[32, 17, 28], n_wait=[6, 16, 0], n_fp=[0, 0, 0], n_a=[4, 2, 3]), "v2", "store"),
    # widest wave block 48, no wait block, fingerprints: the 48-wide tile is full
    "wave48_fp": (dict(n_wave=[48, 33, 40], n_wait=[0, 0, 0], n_fp=[16, 0, 9], n_a=[6, 3, 2], ff=FP), "v2", "store"),
    # dx 224 at the limits: 16 fingerprints, 16 wait inputs, 8 actions next to 2-action agents, an agent without
    # fingerprints, agents without wait inputs
    "limits": (dict(n_wave=[31, 20, 12, 25, 8], n_wait=[16, 0, 6, 0, 6], n_fp=[16, 0, 5, 16, 3], n_a=[8, 2, 2, 5, 3],
                    ff=FP), "v2", "lean"),
}

# one past each kernel limit: (layout kwargs, error text of the construction)
BEYOND = {
    "wave49": (dict(n_wave=[49, 10], n_wait=[0, 0], n_fp=[0, 0], n_a=[3, 2], ft=0), "kernel limits"),
    "fp17": (dict(n_wave=[20, 10], n_wait=[0, 0], n_fp=[17, 3], n_a=[3, 2], ff=FP, ft=0), "kernel limits"),
    "wait17": (dict(n_wave=[20, 10], n_wait=[17, 3], n_fp=[0, 0], n_a=[3, 2]), "kernel limits"),
    "max_na9": (dict(n_wave=[20, 10], n_wait=[4, 3], n_fp=[0, 0], n_a=[9, 2]), "max_na > 8"),
    "dx240": (dict(n_wave=[20, 10], n_wait=[4, 3], n_fp=[4, 0], n_a=[3, 2], fw=144, ff=FP), "dx <= 224"),
}
