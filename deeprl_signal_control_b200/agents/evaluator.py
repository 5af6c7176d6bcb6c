"""`Evaluator`: test-mode evaluation of a trained policy (or the greedy controller) on the device, every test seed at
once — the batched counterpart of reference utils.py:Tester.perform / Evaluator.run (utils.py:195-234, 311-388).

    Evaluator(env, model, output_path, demo=False, policy_type='default', seed=None).run()

`env` is a scenario env (LargeGridEnv, RealNetEnv, ...) built with `n_replicas == env.test_num`: replica k plays the
episode the one-replica env plays after `reset(test_ind=k)` (seed `test_seeds[k]`, test-mode rewards), and in record
mode `output_data()` writes the control / traffic / trip CSVs with the rows, in the order, that the one-replica env
writes when it runs the seeds one after another.  `model` is an IA2C / MA2C wrapper (agents/models.py; only its
parameters `batched.P` and the packed image `batched.Wp` are read), an IQL (`model.name == 'iql'`, LR or DQN; only its
`nets` are read, packed into the evaluator's own parameter vector at the start of every perform_all()) or a greedy
controller (`model.name == 'greedy'`).

Per control step, with no host synchronisation inside the episode: the pi-only forward (tscl_policy_step_pi for the
fused tensor-core widths; the v1 forward or the fc-policy kernels, then tscl_argmax_actions, otherwise), the fp32 Q
forward tscl_q_step (IQL: argmax of q, or the normalised-q sample of IQL.forward(stochastic=True)) or
tsc_greedy_actions; for MA2C the fingerprint is the pi just computed; tsc_step (tsc_step_record in record mode); the
global reward goes into a [T][R] float32 trace.  The evaluator owns every buffer it writes, so a live learner's
parameters, optimiser slot, recurrent states, rollout and counters are left as they were.

`GroupEvaluator` evaluates several agent directories on the same seeds in one process (the reference's `main.py evaluate
--agents`): entries whose simulators would be built identically share one, and the grouped forwards
(tscl_policy_step_pi_g, tscl_q_step_g) serve all their members in one launch per step.
"""
from __future__ import annotations

import ctypes as C
import logging

import numpy as np
import torch

from .. import _lib


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def replica_seeds(env):
    """Replica k plays test episode k: the seed the one-replica env takes after reset(test_ind=k) in test mode (not the
    `seed + r` mapping env.reset uses for n_replicas > 1)."""
    return np.asarray(env.test_seeds, dtype=np.uint64)


def control_frame(actions, greward, ci):
    """Control rows of envs/env.py (the reference's `control_data`): actions [R][T][N] int, greward [R][T] float32;
    replica k is episode k + 1."""
    import pandas as pd
    R, T = greward.shape
    return pd.DataFrame({'episode': np.repeat(np.arange(1, R + 1), T),
                         'time_sec': np.tile(np.arange(1, T + 1) * ci, R),
                         'step': np.tile(np.arange(1, T + 1) * ci / ci, R),
                         'action': [','.join(['%d' % a for a in row]) for row in actions.reshape(R * T, -1)],
                         'reward': greward.reshape(-1).astype(np.float64)})


def traffic_frame(stats):
    """Traffic rows of envs/env.py `_record_traffic`: stats [R][S][8] float32 per simulated second (tsc_step_record
    fields); departed / arrived are per-second differences of the cumulative counters."""
    import pandas as pd
    R, S, _ = stats.shape
    dep, arr = stats[..., 1].astype(np.int64), stats[..., 2].astype(np.int64)
    zero = np.zeros((R, 1), np.int64)
    return pd.DataFrame({'episode': np.repeat(np.arange(1, R + 1), S), 'time_sec': np.tile(np.arange(1, S + 1), R),
                         'number_total_car': stats[..., 0].astype(np.int64).reshape(-1),
                         'number_departed_car': np.diff(dep, axis=1, prepend=zero).reshape(-1),
                         'number_arrived_car': np.diff(arr, axis=1, prepend=zero).reshape(-1),
                         'avg_wait_sec': stats[..., 3].astype(np.float64).reshape(-1),
                         'avg_speed_mps': stats[..., 4].astype(np.float64).reshape(-1),
                         'std_queue': stats[..., 6].astype(np.float64).reshape(-1),
                         'avg_queue': stats[..., 5].astype(np.float64).reshape(-1)})


def trip_frame(trips):
    """Trip rows of envs/env.py `collect_tripinfo`: trips[k] = BatchedSim.trips(k) of episode k + 1."""
    import pandas as pd
    if sum(len(t) for t in trips) == 0:
        return pd.DataFrame([])                               # what the env writes when no vehicle arrived
    ep = np.concatenate([np.full(len(t), k + 1, np.int64) for k, t in enumerate(trips)] + [np.zeros(0, np.int64)])
    rows = np.concatenate([np.asarray(t, np.int64).reshape(-1, 5) for t in trips] + [np.zeros((0, 5), np.int64)])
    dep, arr, route, wsec, wcnt = rows.T
    return pd.DataFrame({'episode': ep, 'id': ['r%d.%d' % (r, d) for r, d in zip(route, dep)],
                         'depart_sec': dep.astype(np.float64), 'arrival_sec': arr.astype(np.float64),
                         'duration_sec': (arr - dep).astype(np.float64), 'wait_step': wcnt,
                         'wait_sec': wsec.astype(np.float64)})


def episode_summary(env, policy_type, mean, std, traffic=None, trip=None):
    """Evaluator.summary of the episodes played on `env`'s test seeds (mean / std: one entry per episode)."""
    out = {'scenario': env.name, 'agent': env.agent, 'policy_type': policy_type,
           'seeds': [int(s) for s in env.test_seeds], 'episode_length_sec': int(env.episode_length_sec),
           'episode_mean_reward': [float(x) for x in mean], 'episode_std_reward': [float(x) for x in std],
           'mean_reward': float(np.mean(mean)), 'std_reward': float(np.std(mean))}
    if traffic is not None:
        out.update(avg_queue=float(traffic.avg_queue.mean()), avg_speed_mps=float(traffic.avg_speed_mps.mean()),
                   avg_wait_sec=float(traffic.avg_wait_sec.mean()))
    if trip is not None:
        ep = trip.episode.values.astype(np.int64) if len(trip) else np.zeros(0, np.int64)
        n = np.bincount(ep, minlength=len(mean) + 1)[1:]
        out.update(trips_per_episode=[int(x) for x in n], mean_trips=float(np.mean(n)))
    return out


class Evaluator:
    def __init__(self, env, model, output_path, demo=False, policy_type='default', seed=None):
        if policy_type not in ('default', 'stochastic', 'deterministic'):
            raise ValueError("policy_type must be 'default', 'stochastic' or 'deterministic' (got %r)" % (policy_type,))
        if env.n_replicas != env.test_num:
            raise ValueError("the evaluator plays every test seed at once: build the env with n_replicas == test_num "
                             "(%d), got %d" % (env.test_num, env.n_replicas))
        self.env, self.model, self.output_path, self.demo = env, model, output_path, demo
        self.policy_type = policy_type
        self.agent = env.agent
        self.seed = int(env.seed if seed is None else seed)
        self.env.train_mode = False
        self.test_num = env.test_num
        sim = env._ensure_sim()
        self.sim, self.R, self.dev = sim, sim.R, sim.device
        net = env._tables
        self.N, self.n_obs, self.max_na = net.n_nodes, net.n_obs, net.max_na
        self.T = int(env.T)
        self.ci = int(env.control_interval_sec)
        name = getattr(model, 'name', None)
        self.greedy = name == 'greedy'
        self.fingerprint = name == 'ma2c'
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.obs = torch.zeros(self.R, self.n_obs, **f32)
        self.act = torch.zeros(self.R, self.N, dtype=torch.int32, device=self.dev)
        self.reward = torch.zeros(self.R, self.N, **f32)
        self.done = torch.zeros(self.R, dtype=torch.uint8, device=self.dev)
        self.trace = torch.zeros(self.T, self.R, **f32)
        self.act_trace = None
        self.stats = None
        self.recorded = None          # (control, traffic, trip) frames written by the last output_data()
        if self.greedy:
            prog = model.greedy_program(net.node_obs_off)
            max_cand, off, idx, act = (int(prog[0]),) + tuple(np.ascontiguousarray(a, np.int32) for a in prog[1:])
            _lib.check(_lib.lib().tsc_set_greedy_program(
                sim._h, C.c_int32(max_cand), off.ctypes.data_as(C.POINTER(C.c_int32)),
                idx.ctypes.data_as(C.POINTER(C.c_int32)), act.ctypes.data_as(C.POINTER(C.c_int32))))
            return
        if name == 'iql':
            self._init_q(model, net)
            return
        b = getattr(model, 'batched', None)
        if b is None or name not in ('ia2c', 'ma2c'):
            raise ValueError("Evaluator: batched evaluation covers the greedy controller, IA2C / MA2C and IQL; %r stays on "
                             "the one-replica protocol" % (name,))
        L = b.lay
        if L.n_obs != self.n_obs or not np.array_equal(L.obs_off, np.asarray(net.node_obs_off[:L.A])):
            raise ValueError("Evaluator: the model's observation layout differs from the env's (build the model with "
                             "obs_off=env node_obs_off)")
        self.b, self.lay = b, L
        if not L.recurrent:
            self.family = 'fc'
        elif not b.use_tc:
            raise ValueError("Evaluator: the fp32 twin forward (use_tc=False) has no batched evaluation path; evaluate the "
                             "tensor-core model")
        else:
            self.family = b.paths.forward          # 'v2' or 'v1' (agents/learner.py:learner_paths)
        self.pi = torch.zeros(self.R, L.A, L.max_na, **f32)
        if self.family == 'v2':            # compact pi-unit state [A][R][h]
            self.c = torch.zeros(L.A, self.R, L.h, **f32); self.h = torch.zeros_like(self.c)
        else:
            self.val = torch.zeros(self.R, L.A, **f32)
            if self.family == 'v1':
                self.c = torch.zeros(L.U, self.R, L.h, **f32); self.h = torch.zeros_like(self.c)
            else:
                self.X = torch.empty(L.U, self.R, L.dx, **f32); self.H = torch.empty(L.U, self.R, L.h, **f32)
        if self.fingerprint:
            u = torch.zeros(self.R, self.N, self.max_na, **f32)
            for i, na in enumerate(L.n_a):
                u[:, i, :na] = 1.0 / int(na)                          # envs/env.py:263-269
            self.fp0 = u

    def _init_q(self, model, net):
        """IQL (agents/models.py): LRQPolicy / DeepQPolicy networks on tscl_q_step."""
        from .layout import QLayout
        off = np.asarray(net.node_obs_off)
        n_s = [int(off[i + 1] - off[i]) for i in range(self.N)]
        if list(model.n_s_ls) != n_s or list(model.n_a_ls) != [int(a) for a in net.n_a_ls]:
            raise ValueError("Evaluator: the model's observation layout differs from the env's (IQL n_s %s / n_a %s, env "
                             "observation widths %s / n_a %s)" % (list(model.n_s_ls), list(model.n_a_ls), n_s,
                                                                  list(net.n_a_ls)))
        self.family = 'q'
        self.qlay = QLayout.from_iql(model, off, self.n_obs, max_na=self.max_na)
        self._qh = C.c_void_p()
        _lib.check(_lib.lib().tscl_q_create(C.byref(self.qlay.as_c()), C.c_int32(self.dev.index or 0), C.byref(self._qh)))
        self.params = torch.zeros(self.qlay.n_params, dtype=torch.float32, device=self.dev)
        self.q = torch.zeros(self.R, self.N, self.max_na, dtype=torch.float32, device=self.dev)
        self.bad = torch.full((1,), -1, dtype=torch.int64, device=self.dev)

    def __del__(self):
        h = getattr(self, '_qh', None)
        if h is not None and h.value:
            _lib.lib().tscl_q_destroy(h)
            self._qh = None

    def _st(self):
        return C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    # ---- one decision for all replicas -----------------------------------------------------------
    def _actions(self, step: int):
        lib = _lib.lib()
        if self.greedy:
            _lib.check(lib.tsc_greedy_actions(self.sim._h, _p(self.obs), _p(self.act), self._st()))
            return None
        if self.family == 'q':
            _lib.check(lib.tscl_q_step(self._qh, _p(self.params), _p(self.obs), C.c_int64(self.R), _p(self.q),
                                       _p(self.act), C.c_int32(int(self.policy_type == 'stochastic')),
                                       C.c_uint64(self.seed), C.c_int64(step), C.c_int64(0), _p(self.bad), self._st()))
            return None
        b, R, done = self.b, self.R, 1 if step == 0 else 0
        argmax = self.policy_type == 'deterministic'
        seed, stp = C.c_uint64(self.seed), C.c_int64(step)
        if self.family == 'v2':
            _lib.check(lib.tscl_policy_step_pi(b._h, _p(b.P), _p(b.Wp), _p(self.obs), C.c_int64(R), _p(self.c), _p(self.h),
                                               _p(self.c), _p(self.h), _p(self.pi), _p(self.act), C.c_int32(int(argmax)),
                                               C.c_int32(done), seed, stp, C.c_int64(0), C.c_int64(0), C.c_int64(0),
                                               self._st()))
            return self.pi
        act = None if argmax else _p(self.act)
        if self.family == 'v1':
            _lib.check(lib.tscl_policy_step(b._h, _p(b.P), _p(b.Wp), _p(self.obs), C.c_int64(R), _p(self.c), _p(self.h),
                                            _p(self.c), _p(self.h), _p(self.pi), _p(self.val), act, C.c_int32(done), seed,
                                            stp, C.c_int64(0), None, C.c_int32(0), self._st()))
        else:
            _lib.check(lib.tscl_fc_embed(b._h, _p(b.P), _p(self.obs), C.c_int64(R), C.c_int64(R), C.c_int64(0), _p(self.X),
                                         self._st()))
            _lib.check(lib.tscl_fc_hidden_fwd(b._h, _p(b.P), _p(self.X), C.c_int64(R), _p(self.H), self._st()))
            _lib.check(lib.tscl_heads(b._h, _p(b.P), _p(self.H), C.c_int64(R), _p(self.pi), _p(self.val), act, seed, stp,
                                      C.c_int64(0), self._st()))
        if argmax:
            _lib.check(lib.tscl_argmax_actions(b._h, _p(self.pi), C.c_int64(R), _p(self.act), self._st()))
        return self.pi

    def _episode(self):
        """All test seeds, one episode each (Tester.perform for every test_ind at once)."""
        env, sim, lib = self.env, self.sim, _lib.lib()
        record = bool(env.is_record)
        sim.reset(replica_seeds(env))
        sim.set_train_mode(False)
        if record:
            sim.set_record(True)
            self.stats = torch.zeros(self.T, self.R, self.ci, 8, dtype=torch.float32, device=self.dev)
            self.act_trace = torch.zeros(self.T, self.R, self.N, dtype=torch.int32, device=self.dev)
        if not self.greedy and self.family in ('v1', 'v2'):
            self.c.zero_(); self.h.zero_()
        fp = self.fp0 if self.fingerprint else None
        sim.observe(fp, obs_out=self.obs)
        for t in range(self.T):
            pi = self._actions(t)
            fp = pi if self.fingerprint else None
            if record:
                _lib.check(lib.tsc_step_record(sim._h, _p(self.act), _p(fp), _p(self.obs), _p(self.reward),
                                               _p(self.trace[t]), _p(self.done), _p(self.stats[t]), self._st()))
                self.act_trace[t].copy_(self.act)
            else:
                _lib.check(lib.tsc_step(sim._h, _p(self.act), _p(fp), _p(self.obs), _p(self.reward), _p(self.trace[t]),
                                        _p(self.done), self._st()))
        env.cur_sec = self.T * self.ci

    # ---- reference interface ----------------------------------------------------------------------
    def perform_all(self):
        """Batched Tester.perform: (mean_reward [R], std_reward [R]) float64, np.mean / np.std of each replica's
        per-step global rewards (utils.py:230-234).  IQL: the model's current weights are packed first (the model itself
        is not written), and with policy_type 'stochastic' a row whose normalised q is not a distribution raises the
        ValueError np.random.choice raises in the reference."""
        q = not self.greedy and self.family == 'q'
        if q:
            self.params.copy_(self.qlay.pack(self.model.nets))
            self.bad.fill_(-1)
        self._episode()
        if q and self.policy_type == 'stochastic':
            key = int(self.bad.item())
            if key != -1:
                r, step, agent = key >> 40, (key >> 16) & 0xFFFFFF, key & 0xFFFF
                raise ValueError('probabilities are not non-negative: q / sum(q) of agent %d at control step %d of test '
                                 'episode %d (seed %d)' % (agent, step, r, int(self.env.test_seeds[r])))
        tr = self.trace.cpu().numpy()
        cols = [np.array(tr[:, k], dtype=np.float64) for k in range(self.R)]
        return np.array([np.mean(c) for c in cols]), np.array([np.std(c) for c in cols])

    def run(self):
        """Evaluator.run (utils.py:376-388): every test seed, then the CSVs when the env records."""
        env = self.env
        env.cur_episode = 0
        if env.is_record:
            env.init_data(True, env.record_stats, self.output_path)
        mean, std = self.perform_all()
        for k in range(self.R):
            logging.info('test %i, avg reward %.2f' % (k, mean[k]))
        env.cur_episode = self.R
        if env.is_record:
            self.output_data()
        return mean, std

    def summary(self, mean, std, traffic=None, trip=None):
        """The quantities of the reference's recorded-evaluation table (BASELINE.md §1): mean and std over episodes of the
        per-episode mean step reward; with the recorded frames also the means of avg_queue / avg_speed_mps /
        avg_wait_sec over all recorded seconds and the completed trips per episode."""
        return episode_summary(self.env, self.policy_type, mean, std, traffic, trip)

    def frames(self):
        """(control, traffic, trip) DataFrames of the last recorded episode set."""
        R, T = self.R, self.T
        control = control_frame(self.act_trace.permute(1, 0, 2).cpu().numpy(), self.trace.t().cpu().numpy(), self.ci)
        traffic = traffic_frame(self.stats.permute(1, 0, 2, 3).reshape(R, T * self.ci, 8).cpu().numpy())
        trip = trip_frame([self.sim.trips(k) for k in range(R)])
        return control, traffic, trip

    def output_data(self):
        """The reference's three CSVs (envs/env.py output_data): <output_path><scenario>_<agent>_{control,traffic,trip}.csv"""
        if not self.env.is_record or self.stats is None:
            logging.error('Evaluator: no record to output!')
            return None
        control, traffic, trip = self.recorded = self.frames()
        base = self.output_path + ('%s_%s_' % (self.env.name, self.env.agent))
        control.to_csv(base + 'control.csv')
        traffic.to_csv(base + 'traffic.csv')
        trip.to_csv(base + 'trip.csv')
        return control, traffic, trip


# ---- several agents at once ---------------------------------------------------------------------------------------------
# the combined replicas of one shared simulator: the recorded per-second statistics alone take T * ci * 32 bytes per
# replica (115 KB at the grid's 720 control steps of 5 s), so 65536 replicas keep the record under 8 GB
MAX_GROUP_REPLICAS = 1 << 16


def entry_model(agent):
    """The model an agent directory's name selects (main.py:179-190, scripts/evaluate.py): 'greedy', 'ia2c', 'ma2c',
    'a2c', 'iqld' -> IQL 'dqn', any other name -> IQL 'lr'."""
    if agent in ('greedy', 'ia2c', 'ma2c', 'a2c'):
        return agent
    return 'dqn' if agent == 'iqld' else 'lr'


def find_checkpoint(model_dir):
    """True when `model_dir` holds a checkpoint the models' load() takes (checkpoint-<step>.npz, or .pt for A2C)."""
    import os
    import re
    return os.path.isdir(model_dir) and any(re.fullmatch(r'checkpoint-\d+\.(npz|pt)', f) for f in os.listdir(model_dir))


def _frozen(v):
    if isinstance(v, np.ndarray):
        return (v.dtype.str, v.shape, v.tobytes())
    if isinstance(v, dict):
        return tuple((k, _frozen(x)) for k, x in sorted(v.items()))
    if isinstance(v, (list, tuple)):
        return tuple(_frozen(x) for x in v)
    return v


def sim_key(env):
    """Equal for two envs whose simulators are built identically: the scenario, the simulator parameters and every net
    table, compared on the built objects.  MA2C leaves out coop_gamma (parameter and observation scale): members that
    differ only there share a simulator through per-replica coop_gamma.  The env seed is not part of the simulator (it
    keys only the policies' sampling)."""
    import dataclasses
    net, par = env._tables, env._params
    ma2c = par.agent == 'ma2c'
    c = par.as_c()
    cfg = tuple((n, getattr(c, n)) for n, _ in type(c)._fields_ if not (ma2c and n == 'coop_gamma'))
    tables = tuple((f.name, _frozen(getattr(net, f.name))) for f in dataclasses.fields(net)
                   if not (ma2c and f.name == 'obs_scale'))
    return env.name, cfg, tables


class GroupEntry:
    """One agent directory of a GroupEvaluator: `label` (its name on the command line), `agent` (the directory's name),
    `model` (entry_model), `output_path`; after the checks `env` (its own one-seed-set env, no simulator), `config`,
    `seed` ([ENV_CONFIG] seed), and `error` when it was skipped.  After run(): mean / std per episode, the three frames
    and `summary`."""

    def __init__(self, agent_dir, model, output_path):
        import os
        self.agent_dir = agent_dir.rstrip('/')
        self.agent = os.path.basename(self.agent_dir)
        self.label = self.agent_dir
        self.model, self.output_path = model, output_path
        self.env = self.config = self.error = None
        self.mean = self.std = self.recorded = self.summary = None


class GroupEvaluator:
    """Several trained agents on the same test seeds in one process: the reference's `main.py evaluate --agents`
    (main.py:158-222) on shared simulators.

        GroupEvaluator(entries, seeds, policy_type='default', policy='lstm').run()

    `entries`: (agent directory, model, output path) triples, model as entry_model gives it.  The constructor only
    checks and groups, on the host: an entry whose directory, config or checkpoint is missing is logged as an error and
    skipped (`skipped`); an `a2c` entry, or a simulator whose combined replicas exceed MAX_GROUP_REPLICAS, is refused
    with a ValueError naming the entry.  Entries whose simulators would be built identically (sim_key) share one
    simulator, len(seeds) consecutive replicas per entry.  Per control step of a shared simulator: one
    tscl_policy_step_pi_g for the v2-family A2C members of one layout, one tscl_q_step_g per IQL layout (LR / DQN),
    tsc_greedy_actions, the v1 / fc A2C members' own forwards on their row slices, and one tsc_step (tsc_step_record).
    Each entry's reward trace, frames and summary are those `Evaluator` gives for its directory alone: member k samples
    with its own [ENV_CONFIG] seed and member-local replica index, ma2c members their own coop_gamma
    (tsc_set_replica_coop_gamma)."""

    def __init__(self, entries, seeds, policy_type='default', policy='lstm', device=0, max_replicas=MAX_GROUP_REPLICAS):
        import configparser
        import glob
        import os
        from ..envs import make_env
        if policy_type not in ('default', 'stochastic', 'deterministic'):
            raise ValueError("policy_type must be 'default', 'stochastic' or 'deterministic' (got %r)" % (policy_type,))
        self.seeds = [int(s) for s in seeds]
        if not self.seeds:
            raise ValueError('GroupEvaluator: no evaluation seeds')
        self.policy_type, self.policy, self.device = policy_type, policy, device
        self.entries = [GroupEntry(d, m, o) for d, m, o in entries]
        for e in self.entries:
            if e.model == 'a2c':
                raise ValueError("%s: batched evaluation covers greedy, ia2c, ma2c and IQL (got agent 'a2c')" % e.label)
        self.skipped = []
        for e in self.entries:
            inis = sorted(glob.glob(os.path.join(e.agent_dir, 'data', '*.ini')))
            if not os.path.isdir(e.agent_dir):
                e.error = 'no agent directory %s' % e.agent_dir
            elif not inis:
                e.error = 'no config under %s/data/' % e.agent_dir
            elif e.model != 'greedy' and not find_checkpoint(os.path.join(e.agent_dir, 'model')):
                e.error = 'no checkpoint under %s/model/' % e.agent_dir
            if e.error:
                logging.error('%s: %s, skipped' % (e.label, e.error))
                self.skipped.append(e)
                continue
            e.config = configparser.ConfigParser()
            e.config.read(inis[0])
            cfg = e.config['ENV_CONFIG']
            cfg['test_seeds'] = ','.join(str(s) for s in self.seeds)
            cfg['agent'] = e.agent
            e.seed = cfg.getint('seed')
            e.env = make_env(cfg, len(self.seeds), e.output_path, device=device)
        self.groups = []                                 # [[entry, ...]] per shared simulator, in entry order
        keys = []
        for e in self.entries:
            if e.error:
                continue
            k = sim_key(e.env)
            if k in keys:
                self.groups[keys.index(k)].append(e)
            else:
                keys.append(k)
                self.groups.append([e])
        for g in self.groups:
            if len(g) * len(self.seeds) > max_replicas:
                raise ValueError('%s: the %d entries sharing its simulator need %d replicas (%d seeds each), more than '
                                 '%d' % (g[-1].label, len(g), len(g) * len(self.seeds), len(self.seeds), max_replicas))

    # ---- device work ----------------------------------------------------------------------------------------------
    def _build_model(self, e):
        import os
        from ..envs import greedy_controller
        from .models import IA2C, IQL, MA2C
        env = e.env
        if e.model == 'greedy':
            return greedy_controller(env)
        mc = e.config['MODEL_CONFIG']
        kw = dict(n_replicas=1, obs_off=env._tables.node_obs_off, policy=self.policy, device=self.device)
        if e.model == 'ma2c':
            m = MA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, env.n_f_ls, 0, mc, **kw)
        elif e.model == 'ia2c':
            m = IA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, 0, mc, **kw)
        else:
            m = IQL(env.n_s_ls, env.n_a_ls, env.n_w_ls, 0, mc, seed=0, model_type=e.model,
                    device=torch.device('cuda', self.device))
        if not m.load(os.path.join(e.agent_dir, 'model') + '/'):
            raise RuntimeError('%s: the checkpoint under %s/model/ does not load' % (e.label, e.agent_dir))
        return m

    def run(self):
        """Every group, one after another; then each entry's CSVs and summary when its env records.  Returns the entries
        that were evaluated."""
        done = []
        for g in self.groups:
            done += _Group(self, g).run()
        return done


def _layout_key(lay):
    return tuple((k, _frozen(v)) for k, v in sorted(vars(lay).items())
                 if isinstance(v, (int, float, bool, str, list, tuple, np.ndarray)))


class _Group:
    """One shared simulator of a GroupEvaluator and its members' forwards."""

    def __init__(self, ge, entries):
        from ..sim import BatchedSim
        self.ge, self.S = ge, len(ge.seeds)
        models = [ge._build_model(e) for e in entries]
        # members ordered by forward family so that each grouped launch covers consecutive rows
        fam = []
        for e, m in zip(entries, models):
            if e.model == 'greedy':
                fam.append(('greedy',))
            elif e.model in ('lr', 'dqn'):
                fam.append(('q', e.model))
            else:
                f = m.batched.paths.forward if m.layout.recurrent else 'fc'
                if f == 'v2':
                    fam.append(('v2', _layout_key(m.layout)))
                elif f in ('v1', 'fc'):
                    fam.append((f, len(fam)))           # own launches
                else:
                    raise ValueError('%s: the fp32 twin forward has no batched evaluation path' % e.label)
        order = sorted(range(len(entries)), key=lambda i: ([f for f in fam].index(fam[i]), i))
        self.entries = [entries[i] for i in order]
        self.models = [models[i] for i in order]
        fams = [fam[i] for i in order]
        K, S = len(self.entries), self.S
        self.R = R = K * S
        self.row0 = [k * S for k in range(K)]
        e0 = self.entries[0]
        self.ma2c = e0.model == 'ma2c'
        cg = [e.env.coop_gamma for e in self.entries] if self.ma2c else None
        base = e0
        if cg is not None and len(set(cg)) > 1:
            # the simulator marks the observation entries it scales only when built with a coop_gamma other than 1
            base = next((e for e in self.entries if e.env.coop_gamma != 1.0), e0)
        else:
            cg = None
        env = base.env
        self.sim = sim = BatchedSim(env._tables, env._params, R, device=ge.device)
        if cg is not None:
            sim.set_replica_coop_gamma(np.repeat(np.asarray(cg, np.float32), S))
        self.dev = sim.device
        net = env._tables
        self.N, self.n_obs, self.max_na = net.n_nodes, net.n_obs, net.max_na
        self.T, self.ci = int(env.T), int(env.control_interval_sec)
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.obs = torch.zeros(R, self.n_obs, **f32)
        self.act = torch.zeros(R, self.N, dtype=torch.int32, device=self.dev)
        self.reward = torch.zeros(R, self.N, **f32)
        self.done = torch.zeros(R, dtype=torch.uint8, device=self.dev)
        self.trace = torch.zeros(self.T, R, **f32)
        self.pi = torch.zeros(R, self.N, self.max_na, **f32)
        self.argmax = ge.policy_type == 'deterministic'
        self.fwd = []                 # (kind, first member, last member + 1, state)
        i = 0
        while i < K:
            j = i
            while j < K and fams[j] == fams[i]:
                j += 1
            self._add_forward(fams[i][0], i, j)
            i = j
        if self.ma2c:
            u = torch.zeros(R, self.N, self.max_na, **f32)
            for a, na in enumerate(net.n_a_ls):
                u[:, a, :na] = 1.0 / int(na)                          # envs/env.py:263-269
            self.fp0 = u

    def _rows(self, i, j):
        S = self.S
        return torch.tensor([(k - i) * S for k in range(i, j + 1)], dtype=torch.int64, device=self.dev)

    def _seeds(self, i, j):
        return torch.tensor(np.array([self.entries[k].seed for k in range(i, j)], dtype=np.uint64).view(np.int64),
                            dtype=torch.int64, device=self.dev)

    def _add_forward(self, kind, i, j):
        from .layout import QLayout
        lib, S, f32 = _lib.lib(), self.S, dict(dtype=torch.float32, device=self.dev)
        n = (j - i) * S
        st = dict(i=i, j=j, n=n)
        if kind == 'greedy':
            prog = self.models[i].greedy_program(self.entries[i].env._tables.node_obs_off)
            max_cand, off, idx, act = (int(prog[0]),) + tuple(np.ascontiguousarray(a, np.int32) for a in prog[1:])
            _lib.check(lib.tsc_set_greedy_program(
                self.sim._h, C.c_int32(max_cand), off.ctypes.data_as(C.POINTER(C.c_int32)),
                idx.ctypes.data_as(C.POINTER(C.c_int32)), act.ctypes.data_as(C.POINTER(C.c_int32))))
        elif kind == 'q':
            m0, net = self.models[i], self.entries[i].env._tables
            qlay = QLayout.from_iql(m0, np.asarray(net.node_obs_off), self.n_obs, max_na=self.max_na)
            h = C.c_void_p()
            _lib.check(lib.tscl_q_create(C.byref(qlay.as_c()), C.c_int32(self.dev.index or 0), C.byref(h)))
            st.update(h=h, qlay=qlay, rows=self._rows(i, j), seeds=self._seeds(i, j),
                      params=torch.stack([qlay.pack(self.models[k].nets).to(self.dev) for k in range(i, j)]).contiguous(),
                      q=torch.zeros(n, self.N, self.max_na, **f32),
                      bad=torch.full((j - i,), -1, dtype=torch.int64, device=self.dev))
        elif kind == 'v2':
            b0, L = self.models[i].batched, self.models[i].layout
            st.update(b=b0, rows=self._rows(i, j), seeds=self._seeds(i, j),
                      P=torch.stack([self.models[k].batched.P for k in range(i, j)]).contiguous(),
                      Wp=torch.stack([self.models[k].batched.Wp for k in range(i, j)]).contiguous(),
                      c=torch.zeros(L.A, n, L.h, **f32), h=torch.zeros(L.A, n, L.h, **f32))
        else:                                           # v1 / fc: one member, its own launches
            b, L = self.models[i].batched, self.models[i].layout
            st.update(b=b, val=torch.zeros(n, L.A, **f32))
            if kind == 'v1':
                st.update(c=torch.zeros(L.U, n, L.h, **f32), h=torch.zeros(L.U, n, L.h, **f32))
            else:
                st.update(X=torch.empty(L.U, n, L.dx, **f32), H=torch.empty(L.U, n, L.h, **f32))
        self.fwd.append((kind, st))

    def __del__(self):
        for kind, st in getattr(self, 'fwd', []):
            if kind == 'q' and st['h'].value:
                _lib.lib().tscl_q_destroy(st['h'])
                st['h'] = C.c_void_p()

    def _st(self):
        return C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    def _actions(self, t):
        lib, done, stp = _lib.lib(), 1 if t == 0 else 0, C.c_int64(t)
        for kind, st in self.fwd:
            r0, n = st['i'] * self.S, st['n']
            obs, pi, act = self.obs[r0:r0 + n], self.pi[r0:r0 + n], self.act[r0:r0 + n]
            if kind == 'greedy':
                _lib.check(lib.tsc_greedy_actions(self.sim._h, _p(self.obs), _p(self.act), self._st()))
            elif kind == 'q':
                _lib.check(lib.tscl_q_step_g(st['h'], _p(st['params']), C.c_int64(st['qlay'].n_params), _p(obs),
                                             C.c_int32(st['j'] - st['i']), _p(st['rows']), C.c_int64(n), _p(st['q']),
                                             _p(act), C.c_int32(int(self.ge.policy_type == 'stochastic')),
                                             _p(st['seeds']), stp, _p(st['bad']), self._st()))
            elif kind == 'v2':
                b = st['b']
                _lib.check(lib.tscl_policy_step_pi_g(
                    b._h, _p(st['P']), C.c_int64(st['P'].shape[1]), _p(st['Wp']), C.c_int64(st['Wp'][0].numel()), _p(obs),
                    C.c_int32(st['j'] - st['i']), _p(st['rows']), C.c_int64(n), _p(st['c']), _p(st['h']), _p(st['c']),
                    _p(st['h']), _p(pi), _p(act), C.c_int32(int(self.argmax)), C.c_int32(done), _p(st['seeds']), stp,
                    self._st()))
            else:
                b, seed = st['b'], C.c_uint64(self.entries[st['i']].seed)
                a = None if self.argmax else _p(act)
                if kind == 'v1':
                    _lib.check(lib.tscl_policy_step(b._h, _p(b.P), _p(b.Wp), _p(obs), C.c_int64(n), _p(st['c']),
                                                    _p(st['h']), _p(st['c']), _p(st['h']), _p(pi), _p(st['val']), a,
                                                    C.c_int32(done), seed, stp, C.c_int64(0), None, C.c_int32(0),
                                                    self._st()))
                else:
                    _lib.check(lib.tscl_fc_embed(b._h, _p(b.P), _p(obs), C.c_int64(n), C.c_int64(n), C.c_int64(0),
                                                 _p(st['X']), self._st()))
                    _lib.check(lib.tscl_fc_hidden_fwd(b._h, _p(b.P), _p(st['X']), C.c_int64(n), _p(st['H']), self._st()))
                    _lib.check(lib.tscl_heads(b._h, _p(b.P), _p(st['H']), C.c_int64(n), _p(pi), _p(st['val']), a, seed,
                                              stp, C.c_int64(0), self._st()))
                if self.argmax:
                    _lib.check(lib.tscl_argmax_actions(b._h, _p(pi), C.c_int64(n), _p(act), self._st()))

    def _episode(self, record):
        sim, lib = self.sim, _lib.lib()
        sim.reset(np.tile(replica_seeds(self.entries[0].env), len(self.entries)))
        sim.set_train_mode(False)
        if record:
            sim.set_record(True)
            self.stats = torch.zeros(self.T, self.R, self.ci, 8, dtype=torch.float32, device=self.dev)
            self.act_trace = torch.zeros(self.T, self.R, self.N, dtype=torch.int32, device=self.dev)
        for kind, st in self.fwd:
            if kind in ('v1', 'v2'):
                st['c'].zero_(); st['h'].zero_()
            elif kind == 'q':
                st['bad'].fill_(-1)
        fp = self.fp0 if self.ma2c else None
        sim.observe(fp, obs_out=self.obs)
        for t in range(self.T):
            self._actions(t)
            fp = self.pi if self.ma2c else None
            if record:
                _lib.check(lib.tsc_step_record(sim._h, _p(self.act), _p(fp), _p(self.obs), _p(self.reward),
                                               _p(self.trace[t]), _p(self.done), _p(self.stats[t]), self._st()))
                self.act_trace[t].copy_(self.act)
            else:
                _lib.check(lib.tsc_step(sim._h, _p(self.act), _p(fp), _p(self.obs), _p(self.reward), _p(self.trace[t]),
                                        _p(self.done), self._st()))

    def _failed_samples(self):
        """{member: message} for the IQL members whose stochastic sample met a q that is not a distribution (the
        ValueError Evaluator.perform_all raises)."""
        out = {}
        if self.ge.policy_type != 'stochastic':
            return out
        for kind, st in self.fwd:
            if kind != 'q':
                continue
            for k, key in enumerate(st['bad'].cpu().numpy().tolist()):
                if key != -1:
                    e = self.entries[st['i'] + k]
                    r, step, agent = key >> 40, (key >> 16) & 0xFFFFFF, key & 0xFFFF
                    out[st['i'] + k] = ('probabilities are not non-negative: q / sum(q) of agent %d at control step %d '
                                        'of test episode %d (seed %d)' % (agent, step, r, int(e.env.test_seeds[r])))
        return out

    def run(self):
        record = all(e.env.is_record for e in self.entries)
        self._episode(record)
        failed = self._failed_samples()
        tr = self.trace.cpu().numpy()
        S, T, done = self.S, self.T, []
        for k, e in enumerate(self.entries):
            if k in failed:
                e.error = failed[k]
                logging.error('%s: %s' % (e.label, e.error))
                continue
            r0 = self.row0[k]
            cols = [np.array(tr[:, r], dtype=np.float64) for r in range(r0, r0 + S)]
            e.mean, e.std = np.array([np.mean(c) for c in cols]), np.array([np.std(c) for c in cols])
            for i in range(S):
                logging.info('%s: test %i, avg reward %.2f' % (e.label, i, e.mean[i]))
            e.env.cur_episode = S
            e.env.cur_sec = T * self.ci
            traffic = trip = None
            if record:
                rows = slice(r0, r0 + S)
                control = control_frame(self.act_trace[:, rows].permute(1, 0, 2).cpu().numpy(),
                                        self.trace[:, rows].t().cpu().numpy(), self.ci)
                traffic = traffic_frame(self.stats[:, rows].permute(1, 0, 2, 3).reshape(S, T * self.ci, 8).cpu().numpy())
                trip = trip_frame([self.sim.trips(r) for r in range(r0, r0 + S)])
                e.recorded = control, traffic, trip
                base = e.output_path + ('%s_%s_' % (e.env.name, e.env.agent))
                control.to_csv(base + 'control.csv')
                traffic.to_csv(base + 'traffic.csv')
                trip.to_csv(base + 'trip.csv')
            e.summary = episode_summary(e.env, self.ge.policy_type, e.mean, e.std, traffic, trip)
            done.append(e)
        return done
