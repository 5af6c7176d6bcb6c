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

Members (`seeds` with K > 1 entries, optionally `member_configs`): a population or sweep of K learners of one layout in
one lock-step of K * R_m replicas, member k on rows [k R_m, (k+1) R_m) of one shared ring [B][K R_m][...], with its own
weights, Adam slots, gradient and (sweep) gamma, max_grad_norm, reward scaling, lr and ε.  Every member keeps the
learner seed (0, as every IQL run), indexes its replicas from 0 and shares the Adam step count and the minibatch
indices, so member k's weights, Adam state, losses and norms are bit-identical to its solo run's (tscl_q_*_g).
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
MAX_MEMBERS = 64                  # members of one grouped launch (QG_MAX, csrc/tsc_q.cu)


_p = _lib.ptr


def ring_bytes(n_replicas: int, buffer_size: int, n_obs: int, n_agents: int) -> int:
    """Device bytes of the replay rings: s and s1 fp32, a int8, r fp32, done u8."""
    return int(n_replicas) * int(buffer_size) * (8 * int(n_obs) + 5 * int(n_agents) + 1)


# the [MODEL_CONFIG] values a member may set for itself; the ring and the networks (batch_size, buffer_size, num_fc,
# num_h) must be the same in every member
MEMBER_KEYS = ('gamma', 'max_grad_norm', 'reward_norm', 'reward_clip')
SHARED_KEYS = ('batch_size', 'buffer_size', 'num_fc', 'num_h')


def check_members(seeds, member_configs, model_config, pg):
    """The member count K of a learner with `seeds` (None: 1) and optional `member_configs`, checked before any device
    work.  Refused with a ValueError: a process group, repeated seeds without member_configs (a population), more than
    MAX_MEMBERS members, a member_configs list of another length, or members whose ring or network differ."""
    if seeds is None:
        if member_configs is not None:
            raise ValueError('member_configs takes `seeds`, one per member')
        return 1
    seeds = [int(s) for s in seeds]
    if not seeds:
        raise ValueError('a population needs at least one seed')
    if pg is not None and len(seeds) > 1:
        raise ValueError('IQL members train in one process: they take no process group')
    if member_configs is None and len(set(seeds)) != len(seeds):
        raise ValueError('population seeds must be distinct (got %s)' % seeds)
    if len(seeds) > MAX_MEMBERS:
        raise ValueError('at most %d members train together (got %d)' % (MAX_MEMBERS, len(seeds)))
    if member_configs is not None:
        if len(member_configs) != len(seeds):
            raise ValueError('a sweep takes one config per seed (got %d configs for %d seeds)'
                             % (len(member_configs), len(seeds)))
        for k, c in enumerate(member_configs):
            for key in SHARED_KEYS:
                a, b = model_config.get(key, fallback=None), c.get(key, fallback=None)
                if a != b and not (a is not None and b is not None and float(a) == float(b)):
                    raise ValueError('[MODEL_CONFIG] %s differs between member 0 (%s) and member %d (%s): the members '
                                     'share one replay ring and one network shape' % (key, a, k, b))
    return len(seeds)


def member_lr_t(lr, t):
    """Each member's Adam step size at step count t, float32: td_round's expression on each member's lr, so the values
    are the solo runs' (whose float the call rounds to float32)."""
    return np.asarray([x * np.sqrt(1.0 - 0.999 ** t) / (1.0 - 0.9 ** t) for x in lr], np.float32)


class BatchedIQL:
    name = 'iql'

    def __init__(self, layout: QLayout, n_replicas: int, model_config, model_type: str, seed: int = 0, device=0,
                 replica0: int = 0, total_replicas: int | None = None, pg=None, seeds=None, member_configs=None):
        """`seeds`: K members (a population), each on n_replicas replicas, each initialised as IQL(seed) is; `seeds` are
        the members' [ENV_CONFIG] seeds and key only their episodes (`BatchedIQLTrainer`), the learner seed stays `seed`.
        `member_configs`: a sweep, one [MODEL_CONFIG] per member, each member's MEMBER_KEYS from its own (seeds may then
        repeat).  One seed is the solo learner."""
        if model_type != layout.model_type:
            raise ValueError("model_type %r differs from the layout's %r" % (model_type, layout.model_type))
        self.K = check_members(seeds, member_configs, model_config, pg)
        self.seeds = None if seeds is None else [int(s) for s in seeds]
        self.lay, self.model_type = layout, model_type
        self.R_m = int(n_replicas)
        self.R, self.replica0 = self.K * self.R_m, int(replica0)
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
        cfgs = member_configs if member_configs is not None else [model_config] * self.K
        # per-member values as the kernels take them: host float32 arrays of K
        self.member_values = {key: np.asarray([c.getfloat(key) or 0.0 for c in cfgs], np.float32) for key in MEMBER_KEYS}
        need = ring_bytes(self.R, self.B, layout.n_obs, layout.A)
        free, _ = torch.cuda.mem_get_info(self.dev)
        if need > free:
            # a ValueError for members: refused, as the other member checks, before any allocation
            raise (MemoryError if self.K == 1 else ValueError)(
                "BatchedIQL: the replay rings need %.2f GB (R=%d x buffer_size=%d x (8 n_obs + 5 A + 1) bytes) but the "
                "device has %.2f GB free" % (need / 1e9, self.R, self.B, free / 1e9))
        self._h = C.c_void_p()
        _lib.check(_lib.lib().tscl_q_create(C.byref(layout.as_c()), self.dev.index or 0, C.byref(self._h)))
        fwd_smem, td_smem = C.c_int64(), C.c_int64()
        _lib.check(_lib.lib().tscl_q_info(self._h, C.byref(fwd_smem), C.byref(td_smem)))
        if td_smem.value == 0:
            # the forward fits but the TD kernel does not: refuse here rather than at the first td_round
            _lib.lib().tscl_q_destroy(self._h)
            self._h = None
            n_wave = layout.n_s - layout.n_w
            i = int(np.argmax(n_wave))
            raise ValueError(
                "BatchedIQL: the TD kernel holds one agent's weights, their gradients and a 64-row tile in shared memory; "
                "with the widest wave block (agent %d: %d wave + %d wait inputs, widths num_fc %d / %d / num_h %d) that "
                "needs %d bytes per CTA but the device has %d.  Evaluation (Evaluator, tscl_q_step) accepts this layout."
                % (i, int(n_wave[i]), int(layout.n_w[i]), layout.n_fc, layout.n_ft, layout.n_h, layout.smem_bytes()[1],
                   torch.cuda.get_device_properties(self.dev).shared_memory_per_block_optin))
        f32 = dict(dtype=torch.float32, device=self.dev)
        p0 = self.initial_params(layout, model_config, model_type, seed)
        self.P = torch.from_numpy(p0 if self.K == 1 else np.stack([p0] * self.K)).to(self.dev)
        self.nets = layout.views(self.P) if self.K == 1 else None
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
        self.idx = torch.zeros(A, self.R_m, self.batch_size, dtype=torch.int32, device=self.dev)
        # flat gradient, then per agent the loss, mean q(s)[a] and mean tq of the round (tscl_q_td's tails)
        pre = () if self.K == 1 else (self.K,)
        self.grad = torch.zeros(pre + (layout.n_params + 3 * A,), **f32)
        self.losses = torch.zeros(pre + (N_ROUNDS, A), **f32)
        self.norms = torch.zeros(pre + (N_ROUNDS, A), **f32)
        self.n_updates = 0                             # backwards that ran (keys the minibatch draws)
        if self.K > 1:
            self.rows = torch.arange(0, self.R + 1, self.R_m, dtype=torch.int64, device=self.dev)
            self._one_scaling = len({(float(n), float(c)) for n, c in zip(self.member_values['reward_norm'],
                                                                         self.member_values['reward_clip'])}) == 1

    def member(self, k: int):
        """Member k as a solo learner (the learner itself without members): its weights, Adam slots, step count, losses
        and norms, for `save`, the `Evaluator`, the summaries and `state_digest`."""
        return self if self.K == 1 else IQLMember(self, k)

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
        return _lib.stream(self.dev)

    @property
    def size(self):
        return min(self.B, self.cum_size)

    @property
    def slot(self):
        """the ring slot the next transition goes to"""
        return self.cum_size % self.B

    # ---- rollout ----------------------------------------------------------------------------------
    def explore(self, obs, eps, step: int):
        """IQL.forward(obs, mode='explore') for all replicas: actions into self.act (int32, for the simulator) and the
        ring slot's s / a.  `step` is the global control step that keys the exploration draws.  With members, `eps` is
        one value per member."""
        k = self.slot
        if self.K > 1:
            e = np.asarray(eps, np.float32)
            _lib.check(_lib.lib().tscl_q_explore_g(
                self._h, _p(self.P), self.lay.n_params, _p(obs), self.K, _p(self.rows), self.R, _p(self.q), _p(self.act),
                e.ctypes.data, self.seed, step, _p(self.s[k]), _p(self.a[k]), self._st()))
            return self.act
        _lib.check(_lib.lib().tscl_q_explore(
            self._h, _p(self.P), _p(obs), self.R, _p(self.q), _p(self.act), eps, self.seed, step, self.replica0,
            _p(self.s[k]), _p(self.a[k]), self._st()))
        return self.act

    def add_transition(self, reward, greward, rew_acc, done: bool):
        """IQL.add_transition: the slot's r (normalised, clipped) and post-step done; s1 was written by the simulator."""
        k = self.slot
        if self.K > 1 and not self._one_scaling:
            mv = self.member_values
            _lib.check(_lib.lib().tscl_q_transition_g(
                self._h, _p(reward), self.K, self.R_m, mv['reward_norm'].ctypes.data, mv['reward_clip'].ctypes.data,
                _p(self.r[k]), _p(greward), _p(rew_acc), _p(self.done[k]), int(done), self._st()))
            self.cum_size += 1
            return
        _lib.check(_lib.lib().tscl_q_transition(
            self._h, _p(reward), self.R, self.reward_norm or 0.0, self.reward_clip or 0.0, _p(self.r[k]), _p(greward),
            _p(rew_acc), _p(self.done[k]), int(done), self._st()))
        self.cum_size += 1

    # ---- update -----------------------------------------------------------------------------------
    def sample(self, rnd: int):
        """This round's minibatch indices idx [A][R_m][batch].  The draws depend on (seed, update, round, replica,
        agent) only, so with members one launch over R_m replicas gives every member its solo run's indices."""
        _lib.check(_lib.lib().tscl_q_sample(
            self._h, self.R_m, self.batch_size, self.size, self.seed, self.n_updates, rnd, self.replica0, _p(self.idx),
            self._st()))
        return self.idx

    def td_round(self, rnd: int, lr: float, idx=None, rec=None):
        """One minibatch round for every agent on the ring entries idx [A][R][batch] (default: this round's draws).
        `rec`: optional float32 [A, 4] device tensor that receives every agent's (loss, mean q, mean tq, pre-clip norm),
        the reference's QPolicy summaries (agents/policies.py:331-338), written by the Adam kernel itself.
        With members: `lr` is one value per member and `rec` a [K, A, 4] tensor (any stride between members)."""
        lib = _lib.lib()
        if idx is None:
            idx = self.sample(rnd)
        if self.K > 1:
            return self._td_round_g(rnd, lr, idx, rec)
        inv_n = 1.0 / (self.batch_size * self.total_replicas)
        _lib.check(lib.tscl_q_td(self._h, _p(self.P), _p(self.s), _p(self.s1), _p(self.a), _p(self.r), _p(self.done),
                                 _p(idx), self.R, self.batch_size, self.gamma, inv_n, _p(self.grad), self._st()))
        if self.pg is not None:
            _dist.allreduce_sum_(self.grad, group=self.pg)
        self.t += 1
        lr_t = lr * np.sqrt(1.0 - 0.999 ** self.t) / (1.0 - 0.9 ** self.t)
        _lib.check(lib.tscl_q_adam(self._h, _p(self.P), _p(self.grad), _p(self.M), _p(self.V), lr_t, self.max_grad_norm,
                                   _p(self.losses[rnd]), _p(self.norms[rnd]), _p(rec), self._st()))

    def _td_round_g(self, rnd, lr, idx, rec):
        lib, mv, n = _lib.lib(), self.member_values, self.lay.n_params
        if len(lr) != self.K:
            raise ValueError('lr takes one value per member (%d, got %d)' % (self.K, len(lr)))
        inv_n = 1.0 / (self.batch_size * self.R_m)
        _lib.check(lib.tscl_q_td_g(self._h, _p(self.P), n, self.K, _p(self.s), _p(self.s1), _p(self.a), _p(self.r),
                                   _p(self.done), _p(idx), self.R_m, self.batch_size, mv['gamma'].ctypes.data, inv_n,
                                   _p(self.grad), self._st()))
        self.t += 1
        lr_t = member_lr_t(lr, self.t)
        _lib.check(lib.tscl_q_adam_g(self._h, self.K, _p(self.P), n, _p(self.grad), _p(self.M), _p(self.V),
                                     lr_t.ctypes.data, mv['max_grad_norm'].ctypes.data, _p(self.losses[:, rnd]),
                                     _p(self.norms[:, rnd]), N_ROUNDS * self.n_agent, _p(rec),
                                     0 if rec is None else rec.stride(0), self._st()))

    def backward(self, lr: float, rec=None) -> bool:
        """IQL.backward after lr = lr_scheduler.get(n_step) (taken by the caller even when this returns False).
        `rec`: optional float32 [N_ROUNDS, A, 4] device tensor; row k receives round k's summaries (td_round)."""
        if self.size < self.batch_size:
            return False
        shape = (N_ROUNDS, self.n_agent, 4) if self.K == 1 else (self.K, N_ROUNDS, self.n_agent, 4)
        if rec is not None and (tuple(rec.shape) != shape or rec.dtype != torch.float32
                                or rec.device != self.dev or not rec.is_contiguous()):
            raise ValueError('rec must be a contiguous float32 %s tensor on %s' % (list(shape), self.dev))
        for k in range(N_ROUNDS):
            if rec is None:
                self.td_round(k, lr)
            else:
                self.td_round(k, lr, rec=rec[k] if self.K == 1 else rec[:, k])
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
        if self.K > 1:
            raise ValueError('a learner with members saves each member: member(k).save(...)')
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


class IQLMember:
    """Member k of a `BatchedIQL` with members as a solo learner: its weights (`nets`, `P`), Adam slots and the shared
    step count, its losses and norms; `save` writes what the solo run's learner writes."""
    name = 'iql'

    def __init__(self, model: BatchedIQL, k: int):
        self._m, self.k = model, int(k)
        self.lay, self.model_type, self.n_agent, self.n_step = model.lay, model.model_type, model.n_agent, model.n_step
        self.n_s_ls, self.n_a_ls, self.n_w_ls = model.n_s_ls, model.n_a_ls, model.n_w_ls
        self.P, self.M, self.V = model.P[self.k], model.M[self.k], model.V[self.k]
        self.nets = model.lay.views(self.P)
        self.losses, self.norms = model.losses[self.k], model.norms[self.k]

    @property
    def t(self):
        return self._m.t

    _prefix = IQL._prefix
    named_weights = IQL.named_weights
    save = BatchedIQL.save
    K = 1


class BatchedIQLTrainer:
    """The reference's IQL explore / backward protocol (utils.py:142-190, 236-250) for R lock-stepped replicas: per control
    step eps = eps_scheduler.get(1), ε-greedy forward, simulator step in train mode straight into the ring slot's s1,
    the slot's r / done; every n_step steps lr = lr_scheduler.get(n_step) and backward; episode ends reset every
    replica with `dist.episode_seeds`.  greward_trace: as in `BatchedTrainer` (row t of the current episode gets step t's
    global reward of every replica; None issues no copy).
    summary_rec: optional float32 [ceil(T_episode / n_step), N_ROUNDS, A, 4] device tensor; the Adam kernel of round k
    of the episode's update j writes every agent's (loss, mean q, mean tq, pre-clip norm) into [j, k], and
    summary_ran[j] says whether update j ran (False while the ring holds fewer than batch_size entries).
    A learner with K > 1 members takes lr_sched / eps_sched as lists of one schedule per member, each called as its solo
    run calls it; it resets member k's replicas with its solo run's seeds (`member_episode_seeds`; seed0 and replica0 are
    not used), keeps summary_rec [ceil(T_episode / n_step), K, N_ROUNDS, A, 4] and appends the list of the K members'
    episode means to `episode_rewards`; `member(k)` is member k's view for the training driver.  `demand`: as in
    `BatchedTrainer`, one NetTables per member whose demand member k's replicas take.  `demand_mix`: as in
    `BatchedTrainer`, the L levels of a mixture, global replica g at level g mod L."""

    def __init__(self, sim, model: BatchedIQL, lr_sched, eps_sched, seed0: int = 12, replica0: int = 0,
                 greward_trace=None, summary_rec=None, demand=None, demand_mix=None):
        from .trainer import _check_rec, _check_trace, set_member_demand, set_mix_demand
        self.K = model.K
        set_member_demand(sim, demand, self.K)
        set_mix_demand(sim, demand_mix, replica0)
        if self.K > 1 and (len(lr_sched) != self.K or len(eps_sched) != self.K):
            raise ValueError('a learner with %d members takes one lr and one ε schedule per member' % self.K)
        self.sim, self.model = sim, model
        self.lr_sched, self.eps_sched = lr_sched, eps_sched
        self.seed0, self.replica0 = int(seed0), int(replica0)
        self.total_replicas = model.total_replicas
        self.T_episode = int(np.ceil(sim.params.episode_length_sec / sim.params.control_interval_sec))
        self.greward_trace = _check_trace(greward_trace, self.T_episode, sim)
        n_upd = -(-self.T_episode // model.n_step)
        self.summary_rec = _check_rec(summary_rec, (n_upd,) + ((self.K,) if self.K > 1 else ()) +
                                      (N_ROUNDS, model.n_agent, 4), sim.device)
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

    def member(self, k: int):
        """Member k's view of this trainer (the trainer itself without members)."""
        from .trainer import MemberTrainer
        return self if self.K == 1 else MemberTrainer(self, k)

    def start_episode(self):
        sim = self.sim
        if self.K > 1:
            from .trainer import member_episode_seeds
            seeds = member_episode_seeds(self.model.seeds, self.episode, self.model.R_m)
        else:
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
        eps = [s.get(1) for s in self.eps_sched] if self.K > 1 else self.eps_sched.get(1)

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
            lr = [s.get(m.n_step) for s in self.lr_sched] if self.K > 1 else self.lr_sched.get(m.n_step)
            if self.summary_rec is None:
                ran = self._timed(self.update_events, lambda: m.backward(lr))
            else:
                j = (self.step_in_episode - 1) // m.n_step
                ran = self._timed(self.update_events, lambda: m.backward(lr, rec=self.summary_rec[j]))
                self.summary_ran[j] = ran
            if ran:
                self.n_updates += 1
        if done:
            if self.K > 1:
                R_m = m.R_m
                self.episode_rewards.append([float((self._rew_acc[k * R_m:(k + 1) * R_m] / self.T_episode).mean())
                                             for k in range(self.K)])
            else:
                self.episode_rewards.append(float((self._rew_acc / self.T_episode).mean()))
            self.start_episode()

    def run(self, n_control_steps: int):
        for _ in range(n_control_steps):
            self.control_step()
