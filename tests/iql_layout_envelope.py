"""Layouts of tests/test_iql_layout_envelope_cpu.py and tests/test_iql_layout_envelope_gpu.py: the shipped scenarios'
IQL agents at the reference's widths (num_fc 128, so num_fc / 4 = 32 wait units, num_h 64), built the way
agents/models.py:IQL and QLayout.from_iql build them, and synthetic layouts at the edges of what the Q kernels accept
(tscl_q_create: widths multiples of 16 up to 128 / 32 / 64, max_na <= 8; the TD kernel's shared memory).

A case is (kind, IQL n_s / n_a / n_w lists, obs_off, n_obs, max_na, model config)."""
import configparser

import numpy as np

from tests.layout_envelope import net_tables

INI = """
[MODEL_CONFIG]
gamma = 0.99
lr_init = 1e-4
lr_decay = constant
epsilon_init = 1.0
epsilon_min = 0.01
epsilon_decay = linear
epsilon_ratio = 0.5
max_grad_norm = 40
batch_size = 20
buffer_size = %d
reward_norm = 1.0
reward_clip = 2.0
num_fc = %d
num_h = %d
"""
FC, H = 128, 64
SPARE = 3                 # observation floats past the last agent's slice that belong to no agent


def model_config(num_fc=FC, num_h=H, buffer_size=1000):
    cp = configparser.ConfigParser()
    cp.read_string(INI % (buffer_size, num_fc, num_h))
    return cp["MODEL_CONFIG"]


class Case:
    def __init__(self, kind, n_s, n_a, n_w, obs_off, n_obs, max_na, num_fc=FC, num_h=H):
        self.kind, self.n_s, self.n_a, self.n_w = kind, [int(x) for x in n_s], [int(x) for x in n_a], [int(x) for x in n_w]
        self.obs_off, self.n_obs, self.max_na = np.asarray(obs_off, np.int64), int(n_obs), int(max_na)
        self.num_fc, self.num_h = num_fc, num_h

    def cfg(self, buffer_size=1000):
        return model_config(self.num_fc, self.num_h, buffer_size)

    def iql(self, seed=0, total_step=0, device="cpu", buffer_size=1000):
        from deeprl_signal_control_b200.agents.models import IQL
        return IQL(self.n_s, self.n_a, self.n_w, total_step, self.cfg(buffer_size), seed=seed, model_type=self.kind,
                   device=device)

    def layout(self, model=None):
        """QLayout.from_iql of the case's IQL (the evaluator's construction; BatchedIQL takes the same layout)"""
        from deeprl_signal_control_b200.agents.layout import QLayout
        return QLayout.from_iql(self.iql() if model is None else model, self.obs_off, self.n_obs, max_na=self.max_na)


def scenario_case(scenario, agent, mini_dir=None):
    """IQL on the scenario's tables as the env hands them to the model: n_s from node_obs_off, the tables' max_na"""
    net = net_tables(scenario, agent, mini_dir)
    off = np.asarray(net.node_obs_off)
    n_s = [int(off[i + 1] - off[i]) for i in range(net.n_nodes)]
    return Case("dqn" if agent == "iqld" else "lr", n_s, net.n_a_ls, net.n_w_ls, off, net.n_obs, net.max_na)


def synthetic_case(n_wave, n_wait, n_a, kind="dqn", num_fc=FC, num_h=H, max_na=None):
    """agents with the given wave / wait blocks, observation slices back to back plus SPARE floats at the end"""
    n_s = [w + t for w, t in zip(n_wave, n_wait)]
    off = np.concatenate([[0], np.cumsum(n_s)])
    return Case(kind, n_s, n_a, n_wait, off, int(off[-1]) + SPARE, max_na or max(n_a), num_fc, num_h)


SCENARIOS = [(s, a) for s in ("large_grid", "real_net", "small_grid", "mini_sumo") for a in ("iqll", "iqld")]

# The widest wave block next to 6 wait inputs whose TD kernel still fits the H100's 232,448 bytes of opt-in shared memory
# at the reference's widths: (324 W + 38856) floats (QLayout.smem_bytes); the GPU test finds it again with tscl_q_info.
TD_WAVE_MAX = 59

EDGES = {
    # num_fc 64 / num_h 32: n_ft = 16, every column loop of the three layers half or a quarter used; mixed wait blocks
    "fc64_h32": dict(n_wave=[20, 13, 30], n_wait=[6, 0, 4], n_a=[5, 3, 2], num_fc=64, num_h=32),
    # the narrowest widths, no wait inputs (num_fc / 4 = 4 would be refused with them)
    "fc16_h16": dict(n_wave=[12, 7, 25], n_wait=[0, 0, 0], n_a=[3, 4, 2], num_fc=16, num_h=16),
    # wait blocks of 16, 0, 3, 0 inputs: per-agent q_fc_0 input widths and zero-length q_fct layers inside the flat vector
    "mixed_wait": dict(n_wave=[22, 17, 9, 30], n_wait=[16, 0, 3, 0], n_a=[4, 3, 5, 2]),
    # 8 actions next to 2-action agents
    "max_na8": dict(n_wave=[14, 20, 9], n_wait=[4, 0, 2], n_a=[8, 2, 2]),
    # observation slices of 15, 27 and 11 floats
    "odd_ns": dict(n_wave=[13, 27, 7], n_wait=[2, 0, 4], n_a=[3, 5, 2]),
    # the widest wave block whose TD layout fits
    "td_wave_max": dict(n_wave=[TD_WAVE_MAX, 21], n_wait=[6, 0], n_a=[4, 3]),
    # LRQPolicy on a wide observation slice
    "lr_wide": dict(n_wave=[200, 37, 120], n_wait=[0, 0, 0], n_a=[5, 2, 8], kind="lr"),
}

# one past each limit: (layout kwargs, error text of the BatchedIQL construction)
WIDTHS = "dqn widths must be multiples of 16"
BEYOND = {
    "fc144": (dict(n_wave=[20, 10], n_wait=[4, 0], n_a=[3, 2], num_fc=144), WIDTHS),
    "h80": (dict(n_wave=[20, 10], n_wait=[4, 0], n_a=[3, 2], num_h=80), WIDTHS),
    "fc96": (dict(n_wave=[20, 10], n_wait=[4, 0], n_a=[3, 2], num_fc=96), WIDTHS),            # n_ft = 24
    "fc32_wait": (dict(n_wave=[20, 10], n_wait=[4, 0], n_a=[3, 2], num_fc=32), WIDTHS),       # n_ft = 8
    "max_na9": (dict(n_wave=[20, 10], n_wait=[4, 3], n_a=[9, 2]), "max_na > 8"),
    # the forward fits, the TD kernel does not: refused by BatchedIQL, accepted for evaluation
    "td_wave_beyond": (dict(n_wave=[TD_WAVE_MAX + 1, 21], n_wait=[6, 0], n_a=[4, 3]), "widest wave block"),
}
# accepted counterpart of fc32_wait: num_fc 32 without wait inputs
FC32_NO_WAIT = dict(n_wave=[20, 10], n_wait=[0, 0], n_a=[3, 2], num_fc=32)

DEFECTS = ("wait block read as wave inputs", "q_fct branch on an agent without a wait block", "done mask dropped",
           "next agent's observation slice")


def agent_batch(lay, P, i, obs, obs1, defect=None):
    """What q_td_ref reads for agent i: (weights, n_w, S, S1, mutate), with planted defect `defect` (None where it does
    not apply to the agent).  P: the flat weight vector (numpy); obs / obs1: [rows][n_obs] observation rows of s / s1.
      wait block read as wave inputs: the wave inputs taken n_w floats further on, so that the wait block is among them;
      q_fct branch on an agent without a wait block: the branch over zero inputs (relu of its bias) and the q_fc_0 rows
      behind it, both read at the agent's offsets into the flat vector, as a kernel that kept n_ft for the agent would;
      done mask dropped: tq = r + gamma max q(s1) for terminal rows too;
      next agent's observation slice: the agent's n_s floats read one slice width further on."""
    P = np.asarray(P, np.float64)
    w = {k: np.array(v) for k, v in lay.views(P)[i].items()}
    o0, n_s, n_w = int(lay.obs_off[i]), int(lay.n_s[i]), int(lay.n_w[i])
    cols, mutate, fct = np.arange(o0, o0 + n_s), None, False
    if defect == "wait block read as wave inputs":
        if n_w == 0:
            return None
        cols = np.concatenate([np.arange(o0 + n_w, o0 + n_s), np.arange(o0 + n_s - n_w, o0 + n_s)])
    elif defect == "q_fct branch on an agent without a wait block":
        if lay.n_ft == 0 or n_w > 0 or i == lay.A - 1:       # the last agent's reads would leave the vector
            return None
        fct = True
    elif defect == "done mask dropped":
        mutate = "no_done"
    elif defect == "next agent's observation slice":
        cols = np.minimum(cols + n_s, lay.n_obs - 1)
    else:
        assert defect is None, defect
    S, S1 = obs[:, cols], obs1[:, cols]
    if fct:
        n_fc, n_ft, n_h = lay.n_fc, lay.n_ft, lay.n_h
        w["q_fct/w"] = np.zeros((1, n_ft))
        w["q_fct/b"] = P[int(lay.off_fct_b[i]):int(lay.off_fct_b[i]) + n_ft]
        o = int(lay.off_fc0_w[i])
        w["q_fc_0/w"] = P[o:o + (n_fc + n_ft) * n_h].reshape(n_fc + n_ft, n_h)
        S, S1 = (np.concatenate([x, np.zeros((x.shape[0], 1))], 1) for x in (S, S1))
        n_w = 1
    return w, n_w, S, S1, mutate


def rel_l2(g, ref):
    g, ref = np.asarray(g, np.float64), np.asarray(ref, np.float64)
    return float(np.sqrt(((g - ref) ** 2).sum() / max((ref ** 2).sum(), 1e-300)))


def moved(a, b, kind):
    """how far round result b is from a, in units of the GPU bounds: (ratio, what moved most).  a, b: q_td_ref outputs
    or the kernel's (loss, grads); gradients compared where the tensor shapes agree"""
    out = [(abs(b["loss"] - a["loss"]) / abs(a["loss"]) / LOSS_BOUND[kind], "loss")]
    for k, g in a["grads"].items():
        if k in b["grads"] and np.shape(b["grads"][k]) == np.shape(g):
            out.append((rel_l2(b["grads"][k], g) / GRAD_BOUND[kind], k))
    return max(out)


# Bounds of one TD round on the device against float64 (tests/test_iql_layout_envelope_gpu.py), per model: rel-L2 of a
# named gradient tensor, and relative error of the loss / mean q / mean tq.  Observed on an H100 80GB HBM3 (700 W): lr
# gradient 2.7e-7 (lr_wide q/b), dqn gradient 1.7e-5 (large_grid q_fct/b: 6000 rows of near-cancelling fp32 terms; the
# synthetic layouts stay below 2e-7), loss / mean q / mean tq 2.7e-7.  Planted defects must move the loss or some named
# gradient by at least 10x these (observed: over 1000x).
GRAD_BOUND = {"lr": 8e-7, "dqn": 5e-5}
LOSS_BOUND = {"lr": 8e-7, "dqn": 8e-7}
