"""Batched IQL training on the device: replay rings, ε-greedy Q forward and a fused fp32 TD / Adam update
(csrc/tsc_q.cu, include/tsc_learn.h tscl_q_*).

Data-parallel IQL (agents/models.py:IQL, the reference's agents/models.py:264-376) for R lock-stepped replicas:
* one flat fp32 weight vector in `QLayout` order shared by every replica and rank, per-agent TF1 Adam state (m, v, t);
* one replay ring per replica, capacity B = buffer_size, shared by the replica's agents (the reference adds the same
  (ob, next_ob, done) to every agent's buffer), slot-major so that one slot is a contiguous [R, n_obs] tensor;
* `backward(lr)`: 10 sequential rounds; in each, every replica draws batch_size distinct ring entries per agent
  (random.sample), and the loss is the mean over batch_size * R_total rows of (q(s)[a] - tq)^2 with
  tq = done ? r : r + gamma max q(s1) (no target network, no gradient through tq), then the per-agent global-norm clip
  and the TF1 Adam step of IQL.td_update.
At R = 1 this is the reference's IQL.backward with another random source.
"""
from __future__ import annotations

import ctypes as C
import logging
import os

import numpy as np
import torch

from .. import _lib
from .. import dist as _dist
from .layout import QLayout
from .models import IQL

N_ROUNDS = 10                     # minibatches per agent per backward (agents/models.py:337-345)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def ring_bytes(n_replicas: int, buffer_size: int, n_obs: int, n_agents: int) -> int:
    """Device bytes of the replay rings: s and s1 fp32, a int8, r fp32, done u8."""
    return int(n_replicas) * int(buffer_size) * (8 * int(n_obs) + 5 * int(n_agents) + 1)


class BatchedIQL:
    name = 'iql'

    def __init__(self, layout: QLayout, n_replicas: int, model_config, model_type: str, seed: int = 0, device=0,
                 replica0: int = 0, total_replicas: int | None = None, pg=None):
        if model_type != layout.model_type:
            raise ValueError("model_type %r differs from the layout's %r" % (model_type, layout.model_type))
        self.lay, self.model_type = layout, model_type
        self.R, self.replica0 = int(n_replicas), int(replica0)
        self.total_replicas = int(total_replicas or n_replicas)
        self.pg, self.seed = pg, int(seed)
        self.dev = torch.device('cuda', device) if isinstance(device, int) else torch.device(device)
        self.n_agent = layout.A
        self.n_s_ls = [int(x) for x in layout.n_s]
        self.n_a_ls = [int(x) for x in layout.n_a]
        self.n_w_ls = [int(x) for x in layout.n_w]
        self.n_step = self.batch_size = model_config.getint('batch_size')
        self.B = int(model_config.getfloat('buffer_size'))
        self.gamma = model_config.getfloat('gamma')
        self.max_grad_norm = model_config.getfloat('max_grad_norm')
        self.reward_norm = model_config.getfloat('reward_norm')
        self.reward_clip = model_config.getfloat('reward_clip')
        need = ring_bytes(self.R, self.B, layout.n_obs, layout.A)
        free, _ = torch.cuda.mem_get_info(self.dev)
        if need > free:
            raise MemoryError("BatchedIQL: the replay rings need %.2f GB (R=%d x buffer_size=%d x (8 n_obs + 5 A + 1) "
                              "bytes) but the device has %.2f GB free" % (need / 1e9, self.R, self.B, free / 1e9))
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.P = torch.from_numpy(self.initial_params(layout, model_config, model_type, seed)).to(self.dev)
        self.nets = layout.views(self.P)
        self.M, self.V = torch.zeros_like(self.P), torch.zeros_like(self.P)
        self.t = 0                                     # Adam step count, the same for every agent
        B, R, A, n_obs = self.B, self.R, layout.A, layout.n_obs
        self.s = torch.empty(B, R, n_obs, **f32)
        self.s1 = torch.empty(B, R, n_obs, **f32)
        self.a = torch.zeros(B, R, A, dtype=torch.int8, device=self.dev)
        self.r = torch.zeros(B, R, A, **f32)
        self.done = torch.zeros(B, R, dtype=torch.uint8, device=self.dev)
        self.cum_size = 0
        self.q = torch.zeros(R, A, layout.max_na, **f32)
        self.act = torch.zeros(R, A, dtype=torch.int32, device=self.dev)
        self.idx = torch.zeros(A, R, self.batch_size, dtype=torch.int32, device=self.dev)
        # flat gradient, then per agent the loss, mean q(s)[a] and mean tq of the round (tscl_q_td's tails)
        self.grad = torch.zeros(layout.n_params + 3 * A, **f32)
        self.losses = torch.zeros(N_ROUNDS, A, **f32)
        self.norms = torch.zeros(N_ROUNDS, A, **f32)
        self.n_updates = 0                             # backwards that ran (keys the minibatch draws)
        self._h = C.c_void_p()
        _lib.check(_lib.lib().tscl_q_create(C.byref(layout.as_c()), C.c_int32(self.dev.index or 0), C.byref(self._h)))

    @staticmethod
    def initial_params(layout: QLayout, model_config, model_type: str, seed: int) -> np.ndarray:
        """The weights IQL(seed) starts from (the same ortho_init draws), packed in the layout's order."""
        m = IQL(list(layout.n_s), list(layout.n_a), list(layout.n_w), 0, model_config, seed=seed, model_type=model_type,
                device='cpu')
        return layout.pack(m.nets).numpy()

    def __del__(self):
        h = getattr(self, '_h', None)
        if h is not None and h.value:
            try:
                _lib.lib().tscl_q_destroy(h)
            except (AttributeError, TypeError):      # interpreter shutdown: the loader is already torn down
                pass
            self._h = None

    def _st(self):
        return C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    @property
    def size(self):
        return min(self.B, self.cum_size)

    @property
    def slot(self):
        """the ring slot the next transition goes to"""
        return self.cum_size % self.B

    # ---- rollout ----------------------------------------------------------------------------------
    def explore(self, obs, eps: float, step: int):
        """IQL.forward(obs, mode='explore') for all replicas: actions into self.act (int32, for the simulator) and the
        ring slot's s / a.  `step` is the global control step that keys the exploration draws."""
        k = self.slot
        _lib.check(_lib.lib().tscl_q_explore(
            self._h, _p(self.P), _p(obs), C.c_int64(self.R), _p(self.q), _p(self.act), C.c_float(eps),
            C.c_uint64(self.seed), C.c_int64(step), C.c_int64(self.replica0), _p(self.s[k]), _p(self.a[k]), self._st()))
        return self.act

    def add_transition(self, reward, greward, rew_acc, done: bool):
        """IQL.add_transition: the slot's r (normalised, clipped) and post-step done; s1 was written by the simulator."""
        k = self.slot
        _lib.check(_lib.lib().tscl_q_transition(
            self._h, _p(reward), C.c_int64(self.R), C.c_float(self.reward_norm or 0.0), C.c_float(self.reward_clip or 0.0),
            _p(self.r[k]), _p(greward), _p(rew_acc), _p(self.done[k]), C.c_int32(int(done)), self._st()))
        self.cum_size += 1

    # ---- update -----------------------------------------------------------------------------------
    def sample(self, rnd: int):
        _lib.check(_lib.lib().tscl_q_sample(
            self._h, C.c_int64(self.R), C.c_int32(self.batch_size), C.c_int32(self.size), C.c_uint64(self.seed),
            C.c_int64(self.n_updates), C.c_int32(rnd), C.c_int64(self.replica0), _p(self.idx), self._st()))
        return self.idx

    def td_round(self, rnd: int, lr: float, idx=None, rec=None):
        """One minibatch round for every agent on the ring entries idx [A][R][batch] (default: this round's draws).
        `rec`: optional float32 [A, 4] device tensor that receives every agent's (loss, mean q, mean tq, pre-clip norm),
        the reference's QPolicy summaries (agents/policies.py:331-338), written by the Adam kernel itself."""
        lib = _lib.lib()
        if idx is None:
            idx = self.sample(rnd)
        inv_n = 1.0 / (self.batch_size * self.total_replicas)
        _lib.check(lib.tscl_q_td(self._h, _p(self.P), _p(self.s), _p(self.s1), _p(self.a), _p(self.r), _p(self.done),
                                 _p(idx), C.c_int64(self.R), C.c_int32(self.batch_size), C.c_float(self.gamma),
                                 C.c_float(inv_n), _p(self.grad), self._st()))
        if self.pg is not None:
            _dist.allreduce_sum_(self.grad, group=self.pg)
        self.t += 1
        lr_t = lr * np.sqrt(1.0 - 0.999 ** self.t) / (1.0 - 0.9 ** self.t)
        _lib.check(lib.tscl_q_adam(self._h, _p(self.P), _p(self.grad), _p(self.M), _p(self.V), C.c_float(lr_t),
                                   C.c_float(self.max_grad_norm), _p(self.losses[rnd]), _p(self.norms[rnd]), _p(rec),
                                   self._st()))

    def backward(self, lr: float, rec=None) -> bool:
        """IQL.backward after lr = lr_scheduler.get(n_step) (taken by the caller even when this returns False).
        `rec`: optional float32 [N_ROUNDS, A, 4] device tensor; row k receives round k's summaries (td_round)."""
        if self.size < self.batch_size:
            return False
        if rec is not None and (tuple(rec.shape) != (N_ROUNDS, self.n_agent, 4) or rec.dtype != torch.float32
                                or rec.device != self.dev or not rec.is_contiguous()):
            raise ValueError('rec must be a contiguous float32 [%d, %d, 4] tensor on %s' % (N_ROUNDS, self.n_agent, self.dev))
        for k in range(N_ROUNDS):
            if rec is None:
                self.td_round(k, lr)
            else:
                self.td_round(k, lr, rec=rec[k])
        self.n_updates += 1
        return True

    def reset(self):
        return

    # ---- checkpoints: IQL's file name and variable names, Adam state under __b200__/ ---------------
    # IQL's variable names (agents/policies.py:343,346,383,386) and their reader; `nets` are views into P
    _prefix = IQL._prefix
    named_weights = IQL.named_weights
    load_named = IQL.load_named

    def save(self, model_dir, global_step):
        from . import checkpoint as ck
        ck.save_npz(os.path.join(model_dir, 'checkpoint-%d.npz' % int(global_step)), self.named_weights(),
                    {'adam_m': self.M.cpu().numpy(), 'adam_v': self.V.cpu().numpy(), 'adam_t': np.int64(self.t),
                     'step': np.int64(global_step)})

    def load(self, model_dir, checkpoint=None):
        from . import checkpoint as ck
        files = os.listdir(model_dir) if os.path.exists(model_dir) else []
        steps = [int(f.split('.')[0].split('-')[1]) for f in files
                 if f.startswith('checkpoint-') and len(f.split('.')[0].split('-')) == 2]
        if checkpoint is None and not steps:
            logging.error('Can not find old checkpoint for %s' % model_dir)
            return False
        path = os.path.join(model_dir, 'checkpoint-%d.npz' % (int(checkpoint) if checkpoint is not None else max(steps)))
        if not os.path.exists(path):
            logging.error('Can not find old checkpoint for %s' % model_dir)
            return False
        named, extra = ck.load_npz(path)
        self.load_named(named)
        if 'adam_m' in extra and extra['adam_m'].shape == tuple(self.M.shape):
            self.M.copy_(torch.from_numpy(extra['adam_m'])); self.V.copy_(torch.from_numpy(extra['adam_v']))
            self.t = int(extra['adam_t'])
        return True


class BatchedIQLTrainer:
    """The reference's IQL explore / backward protocol (utils.py:142-190, 236-250) for R lock-stepped replicas: per control
    step eps = eps_scheduler.get(1), ε-greedy forward, simulator step in train mode straight into the ring slot's s1,
    the slot's r / done; every n_step steps lr = lr_scheduler.get(n_step) and backward; episode ends reset every
    replica with `dist.episode_seeds`.  greward_trace: as in `BatchedTrainer` (row t of the current episode gets step t's
    global reward of every replica; None issues no copy).
    summary_rec: optional float32 [ceil(T_episode / n_step), N_ROUNDS, A, 4] device tensor; the Adam kernel of round k
    of the episode's update j writes every agent's (loss, mean q, mean tq, pre-clip norm) into [j, k], and
    summary_ran[j] says whether update j ran (False while the ring holds fewer than batch_size entries)."""

    def __init__(self, sim, model: BatchedIQL, lr_sched, eps_sched, seed0: int = 12, replica0: int = 0,
                 greward_trace=None, summary_rec=None):
        from .trainer import _check_rec, _check_trace
        self.sim, self.model = sim, model
        self.lr_sched, self.eps_sched = lr_sched, eps_sched
        self.seed0, self.replica0 = int(seed0), int(replica0)
        self.total_replicas = model.total_replicas
        self.T_episode = int(np.ceil(sim.params.episode_length_sec / sim.params.control_interval_sec))
        self.greward_trace = _check_trace(greward_trace, self.T_episode, sim)
        n_upd = -(-self.T_episode // model.n_step)
        self.summary_rec = _check_rec(summary_rec, (n_upd, N_ROUNDS, model.n_agent, 4), sim.device)
        self.summary_ran = np.zeros(n_upd, bool)
        self.episode = 0
        self.episode_rewards = []
        self.n_env_steps = 0
        self.n_updates = 0
        self._since_update = 0        # control steps of the current explore() call (it ends at n_step steps or done)
        self._rew_acc = torch.zeros(sim.R, device=sim.device)
        self.obs0 = torch.zeros(sim.R, sim.net.n_obs, device=sim.device)
        self.sim_events = None        # list of (start, end) CUDA events around the rollout step when timing is on
        self.update_events = None     # same around backward()
        self.start_episode()

    def start_episode(self):
        sim = self.sim
        seeds = _dist.episode_seeds(self.seed0, self.episode, self.replica0, sim.R, max(self.total_replicas, sim.R))
        self.episode += 1
        sim.reset(seeds)
        sim.set_train_mode(True)
        sim.observe(None, obs_out=self.obs0)
        self.obs = self.obs0
        self.step_in_episode = 0
        self._rew_acc.zero_()

    def _timed(self, events, fn):
        if events is None:
            return fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); out = fn(); e1.record()
        events.append((e0, e1))
        return out

    def control_step(self):
        m, sim = self.model, self.sim
        eps = self.eps_sched.get(1)

        def rollout():
            k = m.slot
            act = m.explore(self.obs, eps, self.n_env_steps)
            _, reward, greward, _ = sim.step(act, None, obs_out=m.s1[k])
            if self.greward_trace is not None:
                self.greward_trace[self.step_in_episode].copy_(greward)
            self.step_in_episode += 1
            new_done = self.step_in_episode >= self.T_episode
            m.add_transition(reward, greward, self._rew_acc, new_done)
            self.obs = m.s1[k]
            return new_done

        done = self._timed(self.sim_events, rollout)
        self.n_env_steps += 1
        self._since_update += 1
        if self._since_update == m.n_step or done:
            self._since_update = 0
            lr = self.lr_sched.get(m.n_step)
            if self.summary_rec is None:
                ran = self._timed(self.update_events, lambda: m.backward(lr))
            else:
                j = (self.step_in_episode - 1) // m.n_step
                ran = self._timed(self.update_events, lambda: m.backward(lr, rec=self.summary_rec[j]))
                self.summary_ran[j] = ran
            if ran:
                self.n_updates += 1
        if done:
            self.episode_rewards.append(float((self._rew_acc / self.T_episode).mean()))
            self.start_episode()

    def run(self, n_control_steps: int):
        for _ in range(n_control_steps):
            self.control_step()
