"""Device-resident training loop: the batched counterpart of reference utils.py:Trainer.explore/run.

Per control step (utils.py:146-165): policy/value forward -> fingerprint update (MA2C) -> action
sampling -> env.step -> add_transition; per n_step: bootstrap value, backward (utils.py:186-190,
288-291); per episode: env.reset(), model.reset(), pre-decision done = True (utils.py:277-281).
Everything stays on the GPU: the simulator writes the next observation straight into the
learner's rollout slot and reads actions / fingerprints from the learner's buffers.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from .. import _lib
from .. import dist as _dist
from ..sim import BatchedSim
from .learner import BatchedA2C


def _check_trace(trace, T_episode, sim):
    if trace is not None and (tuple(trace.shape) != (T_episode, sim.R) or trace.dtype != torch.float32
                              or trace.device != sim.device):
        raise ValueError("greward_trace must be a float32 [%d, %d] tensor on %s (got %s %s on %s)"
                         % (T_episode, sim.R, sim.device, tuple(trace.shape), trace.dtype, trace.device))
    return trace


def _check_rec(rec, shape, dev):
    if rec is not None and (tuple(rec.shape) != tuple(shape) or rec.dtype != torch.float32 or rec.device != dev
                            or not rec.is_contiguous()):
        raise ValueError("summary_rec must be a contiguous float32 %s tensor on %s (got %s %s on %s)"
                         % (list(shape), dev, tuple(rec.shape), rec.dtype, rec.device))
    return rec


def member_episode_seeds(seeds, episode: int, n_replicas: int) -> np.ndarray:
    """Reset seeds of a population's K * n_replicas replicas for its `episode`-th episode: member k's block is what its
    solo run draws, episode_seeds(seeds[k], episode, 0, n_replicas, n_replicas).  The simulator's random stream is keyed
    by the reset seed and the simulated second only, so member k's replicas then play the solo run's episodes."""
    return np.concatenate([_dist.episode_seeds(s, episode, 0, n_replicas, n_replicas) for s in seeds])


class MemberTrainer:
    """Population member k of a `BatchedTrainer` as the training driver reads a one-member trainer: its rows of the
    reward trace, its episode means and its summary records.  run() steps the whole population."""

    def __init__(self, trainer, k):
        self._tr, self._k = trainer, int(k)
        R_m = trainer.model.R_m
        self._rows = slice(self._k * R_m, (self._k + 1) * R_m)
        self.T_episode, self.summary_ran = trainer.T_episode, trainer.summary_ran

    def run(self, n_control_steps: int):
        self._tr.run(n_control_steps)

    @property
    def greward_trace(self):
        tr = self._tr.greward_trace
        return None if tr is None else tr[:, self._rows].contiguous()

    @property
    def episode_rewards(self):
        return [e[self._k] for e in self._tr.episode_rewards]

    @property
    def summary_rec(self):
        rec = self._tr.summary_rec
        return None if rec is None else rec[:, self._k]


def schedule_values(sched, n_step: int):
    """The value(s) of a schedule for the next update: a float, an object with `get(n_step)`, or a list of either (one
    per sweep member, each advanced by n_step as its solo run's)."""
    if isinstance(sched, (list, tuple)):
        return [schedule_values(s, n_step) for s in sched]
    return sched.get(n_step) if hasattr(sched, "get") else sched


def set_member_demand(sim, demand, K):
    """Member k's replicas (the k-th block of sim.R / K) take their demand from demand[k] (a list of K NetTables);
    None leaves the simulator's built demand."""
    if demand is None:
        return
    if len(demand) != K:
        raise ValueError("demand takes one net per member (%d, got %d)" % (K, len(demand)))
    sim.set_replica_demand(list(demand), np.repeat(np.arange(K), sim.R // K))


def mix_level_of(replica0, R, L):
    """The demand level of replicas [replica0, replica0 + R) of a run on a mixture of L levels: global replica g runs at
    level g mod L, so that every rank and every 64-replica tile holds every level."""
    return (int(replica0) + np.arange(int(R))) % int(L)


def set_mix_demand(sim, demand_mix, replica0=0):
    """One agent on a mixture of demand levels (a list of L NetTables): this simulator's replica r, global replica
    replica0 + r, takes its demand from demand_mix[(replica0 + r) mod L] (`mix_level_of`); None leaves the simulator's
    built demand."""
    if demand_mix is None:
        return
    sim.set_replica_demand(list(demand_mix), mix_level_of(replica0, sim.R, len(demand_mix)))


class BatchedTrainer:
    def __init__(self, sim: BatchedSim, model: BatchedA2C, agent: str, lr, beta,
                 seed0: int = 12, replica0: int = 0, greward_trace: Optional[torch.Tensor] = None,
                 summary_rec: Optional[torch.Tensor] = None, coop_gamma=None, demand=None, demand_mix=None,
                 imit=None, greedy_program=None):
        """lr / beta: floats (the 'constant' schedules of every shipped A2C config) or objects with the reference's
        `Scheduler.get(n_step)` (agents/utils.py:268-281, agents/models.py:175-176); a schedule advances by n_step per
        update exactly as in the reference (its unit is control steps of ONE environment).
        greward_trace: optional float32 [T_episode, R] device tensor; control_step() copies step t's global reward of
        every replica into row t of the current episode.  None: no copy is issued.
        summary_rec: optional float32 [T_episode / n_step, 4] device tensor; update j of the current episode copies
        agent 0's (policy, value, entropy) loss terms (model.stats[:3]) and pre-clip gradient norm (model.norms[0]) into
        row j with two device copies, so that the summaries of an episode need one read.  None: nothing is copied.
        A population learner (model.K > 1 members of model.R_m replicas) resets member k's replicas with its own seeds
        (`member_episode_seeds`; seed0 and replica0 are not used), keeps [T_episode / n_step, K, 4] records and appends
        the list of the K members' episode means to `episode_rewards`.
        A sweep (a learner with `hparams`) passes lr / beta as lists with one schedule per member (`schedule_values`),
        and `coop_gamma`, one MA2C spatial discount per member: member k's replicas then step with its own
        (BatchedSim.set_replica_coop_gamma), and `demand`, one NetTables per member: member k's replicas then take
        their traffic demand from demand[k] (BatchedSim.set_replica_demand).
        demand_mix: one agent trained on a mixture of demand levels, a list of L NetTables; global replica g (this
        simulator's replica g - replica0) runs at level g mod L (`set_mix_demand`).
        A learner with a teacher (`BatchedA2C(teacher=...)`): every control step labels the student's state into
        model.teach_hist[t] before the simulator step (one tsc_pressure_actions or tsc_greedy_actions launch), and every
        update passes the imitation coefficient `imit` (a float, a schedule, or one per sweep member, as lr / beta) to
        backward().  `greedy_program`: the greedy teacher's table, greedy_controller(env).greedy_program(node_obs_off)
        of the training env, set on the simulator once here.  summary_rec then has a 5th column, agent 0's imitation
        loss (model.stats[3])."""
        set_member_demand(sim, demand, int(getattr(model, "K", 1)))
        set_mix_demand(sim, demand_mix, replica0)
        if coop_gamma is not None:
            K, R_m = int(getattr(model, "K", 1)), sim.R // int(getattr(model, "K", 1))
            if len(coop_gamma) != K:
                raise ValueError("coop_gamma takes one value per member (%d, got %d)" % (K, len(coop_gamma)))
            sim.set_replica_coop_gamma(np.repeat(np.asarray(coop_gamma, np.float32), R_m))
        self.sim, self.model, self.agent = sim, model, agent
        self.lr, self.beta = lr, beta
        self.teacher = getattr(model, "teacher", None)
        if self.teacher is None and (imit is not None or greedy_program is not None):
            raise ValueError("imit / greedy_program need a learner with a teacher (BatchedA2C(teacher=...))")
        if self.teacher is not None and imit is None:
            raise ValueError("a learner with teacher %r needs the imitation coefficient `imit`" % self.teacher)
        self.imit = imit
        if self.teacher == "greedy":
            if greedy_program is None:
                raise ValueError("the greedy teacher needs the training env's greedy_program")
            max_cand, off, idx, act = (int(greedy_program[0]),) + tuple(np.ascontiguousarray(a, np.int32)
                                                                       for a in greedy_program[1:])
            _lib.check(_lib.lib().tsc_set_greedy_program(sim._h, max_cand, off.ctypes.data, idx.ctypes.data,
                                                         act.ctypes.data))
        elif greedy_program is not None:
            raise ValueError("greedy_program is the greedy teacher's (the teacher is %r)" % self.teacher)
        self.seed0, self.replica0 = int(seed0), int(replica0)
        self.total_replicas = int(getattr(model, "total_replicas", sim.R))
        self.K = int(getattr(model, "K", 1))
        self.episode = 0
        self.T_episode = int(np.ceil(sim.params.episode_length_sec / sim.params.control_interval_sec))
        assert self.T_episode % model.T == 0                      # utils.py:121
        self.greward_trace = _check_trace(greward_trace, self.T_episode, sim)
        self.summary_rec = _check_rec(summary_rec, (self.T_episode // model.T,) + ((self.K,) if self.K > 1 else ()) +
                                      (5 if self.teacher else 4,), sim.device)
        self.summary_ran = np.ones(self.T_episode // model.T, bool)       # every A2C update runs
        self.step_in_episode = 0
        self.done = True
        self.episode_rewards = []
        self._rew_acc = torch.zeros(sim.R, device=sim.device)
        self.n_updates = 0
        self.n_env_steps = 0
        self._uniform_fp = None
        self.sim_events = None        # list of (start, end) CUDA events around tsc_step when timing is on
        self.update_events = None     # same around update() (bootstrap forward + backward)
        self.start_episode()

    def member(self, k: int):
        """Population member k's view of this trainer (the trainer itself without a population)."""
        return self if self.K == 1 else MemberTrainer(self, k)

    def start_episode(self):
        sim, m = self.sim, self.model
        # envs/env.py:560 (seed += 1 per episode and environment): disjoint over all (rank, episode) pairs
        if self.K > 1:
            seeds = member_episode_seeds(m.seeds, self.episode, m.R_m)
        else:
            seeds = _dist.episode_seeds(self.seed0, self.episode, self.replica0, sim.R, max(self.total_replicas, sim.R))
        self.episode += 1
        sim.reset(seeds)
        sim.set_train_mode(True)
        m.reset()
        fp = None
        if self.agent == 'ma2c':
            if self._uniform_fp is None:
                n = sim.net
                u = torch.zeros(sim.R, n.n_nodes, n.max_na, device=sim.device)
                for i, na in enumerate(n.n_a_ls):
                    u[:, i, :na] = 1.0 / na                       # envs/env.py:263-269
                self._uniform_fp = u
            fp = self._uniform_fp
        assert m.t == 0
        sim.observe(fp, obs_out=m.obs_slot(0))
        self.step_in_episode = 0
        self.done = True
        self._rew_acc.zero_()

    def control_step(self):
        """One control step of all replicas (utils.py:146-165)."""
        sim, m = self.sim, self.model
        t = m.t
        fused = bool(getattr(m, 'tc_v2', False))      # fused tensor-core forward: one-launch transition hand-over
        pi, val, act = m.forward(m.obs_slot(t), self.done, to_hist=True) if fused else m.forward(m.obs_slot(t), self.done)
        fp = pi if self.agent == 'ma2c' else None                 # env.update_fingerprint(policy)
        if self.teacher is not None:
            self.label(t)
        if self.sim_events is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        _, reward, greward, _ = sim.step(act, fp, obs_out=m.obs_hist[t + 1])
        if self.sim_events is not None:
            e1.record()
            self.sim_events.append((e0, e1))
        if self.greward_trace is not None:
            self.greward_trace[self.step_in_episode].copy_(greward)
        self.step_in_episode += 1
        new_done = self.step_in_episode >= self.T_episode         # lock-step: envs/env.py:577-579
        if fused:
            m.add_transition_device(reward, greward, self._rew_acc, self.done, new_done)
        else:
            m.add_transition(reward, self.done, new_done)
            self._rew_acc.add_(greward)
        self.done = new_done
        self.n_env_steps += 1
        if m.t == m.T:
            self.update()

    def label(self, t: int):
        """The teacher's action for the state the student is in at step t (the one obs_hist[t] describes) into
        teach_hist[t]: max-pressure from the lane counts the last simulator step / observe left, greedy from
        obs_hist[t].  Issued before that step's simulator launch."""
        sim, m = self.sim, self.model
        st = sim._stream()
        if self.teacher == "maxpressure":
            _lib.check(_lib.lib().tsc_pressure_actions(sim._h, _lib.ptr(m.teach_hist[t]), st))
        else:
            _lib.check(_lib.lib().tsc_greedy_actions(sim._h, _lib.ptr(m.obs_hist[t]), _lib.ptr(m.teach_hist[t]), st))

    def _no_teacher(self, what):
        if self.teacher is not None:
            raise ValueError("%s does not label states for a teacher (teacher %r): train with control_step()"
                             % (what, self.teacher))

    def control_step_host(self):
        """Same step with the environment driven through the HOST-buffer C-ABI call (tsc_step_host),
        i.e. the way a reference-style caller holds numpy arrays: actions / fingerprints D2H, env step
        (H2D + kernel + D2H inside), observation / reward H2D into the learner.  Not with a teacher."""
        self._no_teacher("control_step_host")
        sim, m = self.sim, self.model
        t = m.t
        pi, val, act = m.forward(m.obs_slot(t), self.done)
        if not hasattr(self, '_pin_act'):       # page-locked staging for the D2H of actions / fingerprints
            self._pin_act = torch.zeros_like(act, device='cpu').pin_memory()
            self._pin_pi = torch.zeros_like(pi, device='cpu').pin_memory()
        self._pin_act.copy_(act, non_blocking=True)
        if self.agent == 'ma2c':
            self._pin_pi.copy_(pi, non_blocking=True)
        torch.cuda.current_stream(sim.device).synchronize()
        act_h = self._pin_act.numpy()
        fp_h = self._pin_pi.numpy() if self.agent == 'ma2c' else None
        obs_h, rew_h, grew_h, _ = sim.step_host(act_h, fp_h)
        m.obs_hist[t + 1].copy_(torch.from_numpy(obs_h), non_blocking=True)
        reward = torch.from_numpy(rew_h).to(sim.device, non_blocking=True)
        self.step_in_episode += 1
        new_done = self.step_in_episode >= self.T_episode
        m.add_transition(reward, self.done, new_done)
        self._rew_acc.add_(torch.from_numpy(grew_h).to(sim.device, non_blocking=True))
        self.done = new_done
        self.n_env_steps += 1
        if m.t == m.T:
            self.update()

    def control_step_host_pipelined(self, n_parts: int = 2):
        """control_step_host() with the replicas split into `n_parts` ranges, one CUDA stream each: while range k sits on
        the PCIe link (tsc_step_host_range: actions H2D, kernel, observations D2H; then observations H2D into the
        learner), the other ranges run their policy forward / simulator kernels.  Same results as control_step_host():
        ranges are independent and the sampling RNG is keyed by the absolute replica.  The host still receives every
        range's observations / rewards in page-locked numpy buffers before the learner consumes them.  Not with a
        teacher."""
        self._no_teacher("control_step_host_pipelined")
        sim, m = self.sim, self.model
        m._one_reward_scaling("the host-range pipeline")
        R, A, L = sim.R, m.lay.A, m.lay
        lib = _lib.lib()
        ma2c = self.agent == 'ma2c'
        if not hasattr(self, '_pp'):
            n_parts = max(1, min(n_parts, R))
            bounds = [R * k // n_parts for k in range(n_parts + 1)]
            pin = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype).pin_memory()
            pp = dict(primed=False, act=pin(R, A, dtype=torch.int32), pi=pin(R, A, L.max_na), obs=pin(R, sim.net.n_obs),
                      rew=pin(R, A), grew=pin(R), done=pin(R, dtype=torch.uint8),
                      rew_stage=torch.zeros(R, A, device=m.dev), grew_stage=torch.zeros(R, device=m.dev), parts=[])
            at = lambda x, r0, per_row: x.data_ptr() + r0 * per_row * x.element_size()
            for k in range(n_parts):        # raw pointers of every range's slices: the per-step loop is host-issue-bound
                r0, n = bounds[k], bounds[k + 1] - bounds[k]
                st = torch.cuda.Stream(device=sim.device)
                pp['parts'].append(dict(
                    r0=r0, n=n, stream=st, sth=st.cuda_stream, ev=torch.cuda.Event(),
                    act_h=at(pp['act'], r0, A), pi_h=at(pp['pi'], r0, A * L.max_na) if ma2c else None,
                    obs_h=at(pp['obs'], r0, sim.net.n_obs), rew_h=at(pp['rew'], r0, A), grew_h=at(pp['grew'], r0, 1),
                    done_h=at(pp['done'], r0, 1), rew_stage=at(pp['rew_stage'], r0, A),
                    grew_stage=at(pp['grew_stage'], r0, 1), rew_acc=at(self._rew_acc, r0, 1)))
            self._pp = pp
        pp = self._pp

        def issue_forward(p, t, nf, done):
            pi, val, act = m.forward_range(p['r0'], p['n'], done, t, nf, stream=p['sth'], to_hist=True)
            _lib.check(lib.tscl_memcpy_async(m._h, p['act_h'], act.data_ptr(), p['n'] * A * 4, 2, p['sth']))
            if ma2c:
                _lib.check(lib.tscl_memcpy_async(m._h, p['pi_h'], pi.data_ptr(), p['n'] * A * L.max_na * 4, 2,
                                                 p['sth']))
            p['ev'].record(p['stream'])

        if not pp['primed']:
            cur = torch.cuda.current_stream(sim.device)
            for p in pp['parts']:
                p['stream'].wait_stream(cur)
                issue_forward(p, m.t, m.n_forward, self.done)
            m.end_forward_ranges()
            pp['primed'] = True
        t = m.t
        self.step_in_episode += 1
        new_done = self.step_in_episode >= self.T_episode
        boundary = (t + 1 == m.T)                       # an update (and possibly an episode end) follows this step
        n_obs = sim.net.n_obs
        for p in pp['parts']:                           # every range's env step is enqueued as soon as its actions are here
            p['ev'].synchronize()                       # the host holds this range's actions / fingerprints
            _lib.check(lib.tsc_step_host_range_async(sim._h, p['r0'], p['n'], p['act_h'], p['pi_h'], p['obs_h'],
                                                     p['rew_h'], p['grew_h'], p['done_h'], p['sth']))
        obs_next, rew_t = m.obs_hist[t + 1], m.rew_hist[t]
        for p in pp['parts']:
            r0, n = p['r0'], p['n']
            p['stream'].synchronize()                   # the host holds this range's observations / rewards ...
            # ... and hands them to the learner: obs -> rollout slot t+1, reward -> normalised / clipped slot t, episode sum
            _lib.check(lib.tscl_host_transition(
                m._h, p['obs_h'], obs_next.data_ptr() + r0 * n_obs * 4, n * n_obs, p['rew_h'], p['rew_stage'],
                rew_t.data_ptr() + r0 * A * 4, n * A, m.reward_norm or 0.0, m.reward_clip or 0.0, p['grew_h'],
                p['grew_stage'], p['rew_acc'], n, p['sth']))
            if not boundary:
                issue_forward(p, t + 1, m.n_forward, False)
        m.end_transition_ranges(self.done, new_done)
        self.done = new_done
        self.n_env_steps += 1
        if not boundary:
            m.end_forward_ranges()
        else:
            cur = torch.cuda.current_stream(sim.device)
            for p in pp['parts']:
                cur.wait_stream(p['stream'])
            pp['primed'] = False
            self.update()

    def update(self):
        m = self.model
        if self.update_events is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        self._update()
        if self.update_events is not None:
            e1.record()
            self.update_events.append((e0, e1))

    def _update(self):
        m = self.model
        boot = None
        if not self.done:
            _, boot, _ = m.forward(m.obs_slot(m.T), False, out_type='v')    # utils.py:190
        if self.teacher is None:
            m.backward(boot, schedule_values(self.lr, m.T), schedule_values(self.beta, m.T))
        else:
            m.backward(boot, schedule_values(self.lr, m.T), schedule_values(self.beta, m.T),
                       schedule_values(self.imit, m.T))
        if self.summary_rec is not None:
            j = self.step_in_episode // m.T - 1
            self.summary_rec[j, ..., :3].copy_(m.stats[..., :3])
            self.summary_rec[j, ..., 3:4].copy_(m.norms[..., :1])
            if self.teacher is not None:
                self.summary_rec[j, ..., 4:].copy_(m.stats[..., 3:4])
        self.n_updates += 1
        if self.done and self.K > 1:
            R_m = m.R_m
            self.episode_rewards.append([float((self._rew_acc[k * R_m:(k + 1) * R_m] / self.T_episode).mean())
                                         for k in range(self.K)])
            self.start_episode()
        elif self.done:
            self.episode_rewards.append(float((self._rew_acc / self.T_episode).mean()))   # utils.py:296-305
            self.start_episode()

    def run(self, n_control_steps: int):
        for _ in range(n_control_steps):
            self.control_step()
