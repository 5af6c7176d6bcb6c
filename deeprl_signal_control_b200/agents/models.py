"""IA2C / MA2C with the reference's constructor and method names (agents/models.py:132-261).

    IA2C(n_s_ls, n_a_ls, n_w_ls, total_step, model_config, seed=0)
    MA2C(n_s_ls, n_a_ls, n_w_ls, n_f_ls, total_step, model_config, seed=0)
    forward(obs, done, out_type='pv'), backward(R_ls, summary_writer=None, global_step=None) (the writer receives agent
    0's loss terms and gradient norm, agents/policies.py:62-72),
    add_transition(obs, actions, rewards, values, done), reset(), save(dir, step), load(dir, checkpoint)
    attributes n_step, n_agent, sess (None: there is no TF session), policy_ls is not provided.

They are thin hosts over `BatchedA2C` (hand-written CUDA kernels); with `n_replicas == 1` the
methods take and return the reference's Python lists / numpy arrays, so `utils.py:Trainer` drives
them unchanged.  `batched` exposes the device-resident learner for R > 1.
"""
from __future__ import annotations

import logging
import os
from typing import List, Optional

import numpy as np
import torch

from .layout import PolicyLayout
from .learner import BatchedA2C
from .utils import Scheduler


def a2c_schedulers(model_config, total_step):
    """(lr_scheduler, beta_scheduler) of IA2C / MA2C (agents/models.py:53-69): lr decays over total_step, the entropy
    coefficient over total_step * entropy_ratio, each 'constant' or 'linear'."""
    lr_init = model_config.getfloat('lr_init')
    lr_decay = model_config.get('lr_decay')
    beta_init = model_config.getfloat('entropy_coef_init')
    beta_decay = model_config.get('entropy_decay')
    if lr_decay == 'constant':
        lr = Scheduler(lr_init, decay=lr_decay)
    else:
        lr = Scheduler(lr_init, model_config.getfloat('LR_MIN'), total_step, decay=lr_decay)
    if beta_decay == 'constant':
        beta = Scheduler(beta_init, decay=beta_decay)
    else:
        beta = Scheduler(beta_init, model_config.getfloat('ENTROPY_COEF_MIN'),
                         total_step * model_config.getfloat('ENTROPY_RATIO'), decay=beta_decay)
    return lr, beta


# [MODEL_CONFIG] keys of imitation (learner.py's module docstring): `teacher = maxpressure | greedy` and the schedule of
# the imitation coefficient lam, which may differ between the members of a sweep
IMITATION_KEYS = ('imitation_coef_init', 'imitation_decay', 'imitation_coef_min', 'imitation_ratio')
IMITATION_DECAYS = ('constant', 'linear')


def check_imitation(model_config, agent):
    """The teacher of an agent's [MODEL_CONFIG] (None without one), every imitation key checked; raises ValueError
    naming the key: an unknown teacher (or a controller that has no action labels), imitation keys without a teacher, a
    teacher without imitation_coef_init, an imitation_decay other than constant / linear, an imitation_coef_init or
    imitation_coef_min that is negative or not finite, an imitation_ratio that is not finite and > 0, and a teacher for
    an IQL agent (iqll / iqld).  Reads nothing but the section: call it before any directory or device work."""
    from .learner import check_imit, check_teacher
    teacher = model_config.get('teacher', fallback=None)
    given = [k for k in IMITATION_KEYS if model_config.get(k, fallback=None) is not None]
    if teacher is None:
        if given:
            raise ValueError('[MODEL_CONFIG] %s: imitation keys need a teacher (teacher = maxpressure | greedy)'
                             % ', '.join(given))
        return None
    try:
        check_teacher(teacher)
    except ValueError as e:
        raise ValueError('[MODEL_CONFIG] teacher: %s' % e)
    if agent not in ('ia2c', 'ma2c'):
        raise ValueError('[MODEL_CONFIG] teacher = %s: imitation trains the A2C agents (ia2c, ma2c), not %r (IQL with '
                         'demonstrations is not built)' % (teacher, agent))
    if 'imitation_coef_init' not in given:
        raise ValueError('[MODEL_CONFIG] imitation_coef_init is required with teacher = %s' % teacher)
    decay = model_config.get('imitation_decay', fallback='constant')
    if decay not in IMITATION_DECAYS:
        raise ValueError('[MODEL_CONFIG] imitation_decay must be one of %s (got %r)' % (', '.join(IMITATION_DECAYS), decay))
    for key in ('imitation_coef_init', 'imitation_coef_min'):
        try:
            check_imit(model_config.get(key, fallback='0'), key)
        except ValueError as e:
            raise ValueError('[MODEL_CONFIG] %s' % e)
    ratio = model_config.getfloat('imitation_ratio', fallback=1.0)
    if not np.isfinite(ratio) or ratio <= 0:
        raise ValueError('[MODEL_CONFIG] imitation_ratio must be finite and > 0 (got %r)' % ratio)
    return teacher


def imitation_scheduler(model_config, total_step):
    """The schedule of the imitation coefficient lam (a `Scheduler`, as the entropy coefficient's): imitation_coef_init,
    'constant', or 'linear' down to imitation_coef_min (default 0) over total_step * imitation_ratio (default 1)."""
    lam0 = model_config.getfloat('imitation_coef_init')
    decay = model_config.get('imitation_decay', fallback='constant')
    if decay == 'constant':
        return Scheduler(lam0, decay=decay)
    return Scheduler(lam0, model_config.getfloat('imitation_coef_min', fallback=0.0),
                     total_step * model_config.getfloat('imitation_ratio', fallback=1.0), decay=decay)


def a2c_hparams(model_config):
    """The `BatchedA2C` values of one [MODEL_CONFIG] section, keyed by learner.SWEEP_KEYS."""
    return dict(gamma=model_config.getfloat('gamma'), v_coef=model_config.getfloat('value_coef'),
                max_grad_norm=model_config.getfloat('max_grad_norm'), alpha=model_config.getfloat('rmsp_alpha'),
                eps=model_config.getfloat('rmsp_epsilon'), reward_norm=model_config.getfloat('reward_norm'),
                reward_clip=model_config.getfloat('reward_clip'))


class IA2C:
    name = 'ia2c'

    def __init__(self, n_s_ls, n_a_ls, n_w_ls, total_step, model_config, seed=0, n_f_ls=None,
                 n_replicas=1, device=0, obs_off=None, policy='lstm', seeds=None, member_configs=None,
                 deterministic=False, **learner_kw):
        """policy='lstm': LstmACPolicy / FPLstmACPolicy, what the reference builds (agents/models.py:40-51);
        policy='fc': FcACPolicy (agents/policies.py:214-256), the FC variant of BASELINE config 2.
        seeds: a population of len(seeds) members, n_replicas each, member k initialised from seeds[k] (`BatchedA2C`;
        LSTM policy only); `members()` gives each as a solo model.
        member_configs: a sweep, one [MODEL_CONFIG] section per seed (model_config is member 0's): member k takes its
        learner values (`a2c_hparams`) and its lr / beta schedules (`lr_schedulers[k]`, `beta_schedulers[k]`) from
        member_configs[k]; seeds may then repeat.
        deterministic: the update adds its gradients in a fixed order, so equal runs give equal bits
        (`BatchedA2C(deterministic=True)`; LSTM policy only)."""
        if seeds is not None and len(seeds) > 1 and policy == 'fc':
            raise ValueError("a population trains the LSTM policy only (got policy='fc')")
        if deterministic:
            if policy == 'fc':
                raise ValueError("deterministic=True needs the LSTM policy's lean update (got policy='fc')")
            learner_kw['deterministic'] = True
        if member_configs is not None:
            if seeds is None or len(member_configs) != len(seeds):
                raise ValueError("a sweep takes one seed per member config")
            learner_kw['hparams'] = [a2c_hparams(c) for c in member_configs]
        if seeds is not None:
            learner_kw['seeds'] = seeds
            seed = int(seeds[0])
        # imitation of a signal controller (learner.py's module docstring): refused by key before any device work
        self.teacher = check_imitation(model_config, self.name)
        if self.teacher:
            learner_kw['teacher'] = self.teacher
        self.n_agent = len(n_s_ls)
        self._pre_done = False
        self.reward_clip = model_config.getfloat('reward_clip')
        self.reward_norm = model_config.getfloat('reward_norm')
        self.n_s_ls, self.n_a_ls, self.n_w_ls = list(n_s_ls), list(n_a_ls), list(n_w_ls)
        self.n_f_ls = list(n_f_ls) if n_f_ls is not None else [0] * self.n_agent
        self.n_step = model_config.getint('batch_size')
        self.sess = None
        self.total_step = total_step
        self.policy = policy
        if obs_off is None:
            obs_off = np.concatenate([[0], np.cumsum(self.n_s_ls)])
        n_obs = int(obs_off[self.n_agent]) if len(obs_off) > self.n_agent else int(np.sum(self.n_s_ls))
        ff = model_config.getint('num_fp') if self.name == 'ma2c' else 0
        self.layout = PolicyLayout(self.n_s_ls, self.n_a_ls, self.n_w_ls, self.n_f_ls, obs_off, n_obs,
                                   fw=model_config.getint('num_fw'), ft=model_config.getint('num_ft'), ff=ff,
                                   h=model_config.getint('num_lstm'), recurrent=(policy != 'fc'))
        if policy == 'fc':
            from .learner_fc import BatchedFcA2C as _Learner
        else:
            _Learner = BatchedA2C
        self.batched = _Learner(
            self.layout, n_replicas, self.n_step, gamma=model_config.getfloat('gamma'),
            v_coef=model_config.getfloat('value_coef'), max_grad_norm=model_config.getfloat('max_grad_norm'),
            alpha=model_config.getfloat('rmsp_alpha'), eps=model_config.getfloat('rmsp_epsilon'),
            reward_norm=self.reward_norm, reward_clip=self.reward_clip, seed=seed, device=device, **learner_kw)
        if total_step:
            self.lr_scheduler, self.beta_scheduler = a2c_schedulers(model_config, total_step)
            if member_configs is not None:
                self.lr_schedulers, self.beta_schedulers = (
                    list(s) for s in zip(*(a2c_schedulers(c, total_step) for c in member_configs)))
            if self.teacher:
                self.imit_scheduler = imitation_scheduler(model_config, total_step)
                if member_configs is not None:
                    self.imit_schedulers = [imitation_scheduler(c, total_step) for c in member_configs]
        self._rng = np.random.RandomState(seed)
        self._obs_dev = torch.zeros(n_replicas, n_obs, device=self.batched.dev)

    # ---- reference protocol (lists in / lists out, one replica) ---------------------------------
    def _pack(self, obs: List[np.ndarray]) -> torch.Tensor:
        row = np.concatenate([np.asarray(o, np.float32) for o in obs])
        self._obs_dev[0, :row.shape[0]].copy_(torch.from_numpy(row))
        return self._obs_dev

    def forward(self, obs, done, out_type='pv'):
        b = self.batched
        slot = b.obs_slot() if ('p' in out_type and b.t < b.T) else self._obs_dev
        slot.copy_(self._pack(obs))
        if 'p' in out_type:
            self._pre_done = bool(done)     # the pre-decision done of this step (utils.py:279-281, agents/utils.py:226)
        pi, val, _ = b.forward(slot, bool(done), out_type, sample=False)
        pol = [pi[0, i, :self.n_a_ls[i]].cpu().numpy() for i in range(self.n_agent)] if 'p' in out_type else None
        vals = [float(v) for v in val[0].cpu().numpy()] if 'v' in out_type else None
        if len(out_type) == 1:
            return pol if out_type == 'p' else vals
        return pol, vals

    def add_transition(self, obs, actions, rewards, values, done):
        b = self.batched
        dev = b.dev
        act = torch.tensor(np.asarray(actions, np.int32).reshape(1, -1), device=dev)
        val = torch.tensor(np.asarray(values, np.float32).reshape(1, -1), device=dev)
        rew = torch.tensor(np.asarray(rewards, np.float32).reshape(1, -1) * np.ones((1, self.n_agent), np.float32),
                           device=dev)
        # the observation of step t is the one the preceding forward('p') consumed (reference: the caller passes the
        # same `ob` to forward and to add_transition, utils.py:148,165); keep the slot authoritative but verify it
        row = np.concatenate([np.asarray(o, np.float32) for o in obs])
        if not np.array_equal(b.obs_slot()[0, :row.shape[0]].cpu().numpy(), row):
            b.obs_slot()[0, :row.shape[0]].copy_(torch.from_numpy(row))
            b._acts_ok[b.t] = False         # stored activations belong to another observation: recompute in backward
        b.add_transition(rew, self._pre_done, bool(done), act=act, val=val)

    def backward(self, R_ls, summary_writer=None, global_step=None):
        cur_lr = self.lr_scheduler.get(self.n_step)
        cur_beta = self.beta_scheduler.get(self.n_step)
        boot = torch.tensor(np.asarray(R_ls, np.float32).reshape(1, -1), device=self.batched.dev)
        self.batched.backward(boot, cur_lr, cur_beta)
        if summary_writer is not None:
            # agents/policies.py:62-72: agent 0's loss terms and pre-clip gradient norm at global_step; any writer with
            # add_scalar(tag, value, step) (agents/summary.py:SummaryWriter, torch.utils.tensorboard) will do
            from .summary import a2c_values, summary_name
            b = self.batched
            rec = torch.cat([b.stats[:3], b.norms[:1]]).cpu().numpy()
            for tag, v in a2c_values(summary_name(self.name, self.policy), rec).items():
                summary_writer.add_scalar(tag, float(v), global_step)

    def reset(self):
        self.batched.reset()

    def members(self):
        """One solo model per population member (itself without a population): name, layout, n_step and the member's
        learner view as `batched`, for `save`, the `Evaluator` and the summaries."""
        b = self.batched
        if getattr(b, 'K', 1) == 1:
            return [self]
        return [A2CMember(self, b.member(k)) for k in range(b.K)]

    # ---- checkpoints: reference file-name convention and VARIABLE NAMES (agents/models.py:83-108, checkpoint.py) ---
    def save(self, model_dir, global_step):
        """`checkpoint-<step>.npz` keyed by the reference's TF variable names (`<policy>_<i>a/pi_fcw/w`, ...); the
        RMSProp slot travels under `__b200__/` so that our own runs can resume (the reference's Saver does not store it)."""
        from . import checkpoint as ck
        b = self.batched
        named = ck.export_named(self.layout, b.P.cpu().numpy())
        ck.save_npz(os.path.join(model_dir, 'checkpoint-%d.npz' % int(global_step)), named,
                    {'rms': b.MS.cpu().numpy(), 'step': np.int64(global_step), 'name': np.array(self.name)})

    def load(self, model_dir, checkpoint=None):
        from . import checkpoint as ck
        save_file, save_step = None, 0
        if os.path.exists(model_dir):
            if checkpoint is None:
                for file in os.listdir(model_dir):
                    if file.startswith('checkpoint'):
                        tokens = file.split('.')[0].split('-')
                        if len(tokens) != 2:
                            continue
                        if int(tokens[1]) >= save_step:
                            save_file, save_step = 'checkpoint-%d' % int(tokens[1]), int(tokens[1])
            else:
                save_file = 'checkpoint-%d' % int(checkpoint)
        base = os.path.join(model_dir, save_file) if save_file is not None else None
        if base is not None and os.path.exists(base + '.npz'):
            named, extra = ck.load_npz(base + '.npz')
            b = self.batched
            b.P.copy_(torch.from_numpy(ck.import_named(self.layout, named)))
            if 'rms' in extra and extra['rms'].shape == tuple(b.MS.shape):
                b.MS.copy_(torch.from_numpy(extra['rms']))
            b.pack_weights()
            logging.info('Checkpoint loaded: %s' % save_file)
            return True
        if base is not None and os.path.exists(base + '.pt'):          # round-1 format
            c = torch.load(base + '.pt')
            self.batched.P.copy_(c['params']); self.batched.MS.copy_(c['rms'])
            self.batched.pack_weights()
            logging.info('Checkpoint loaded: %s' % save_file)
            return True
        logging.error('Can not find old checkpoint for %s' % model_dir)
        return False


class A2CMember:
    """Population member k of an IA2C / MA2C as a solo model: `batched` is the learner's member view."""

    def __init__(self, model, batched):
        self.name, self.policy, self.layout, self.n_agent = model.name, model.policy, model.layout, model.n_agent
        self.n_s_ls, self.n_a_ls, self.n_step = model.n_s_ls, model.n_a_ls, model.n_step
        self.batched = batched

    save = IA2C.save


class MA2C(IA2C):
    name = 'ma2c'

    def __init__(self, n_s_ls, n_a_ls, n_w_ls, n_f_ls, total_step, model_config, seed=0, **kw):
        super().__init__(n_s_ls, n_a_ls, n_w_ls, total_step, model_config, seed=seed, n_f_ls=n_f_ls, **kw)


def iql_schedulers(model_config, total_step):
    """(lr_scheduler, eps_scheduler) of IQL (agents/models.py:305-321): lr decays over total_step, ε over
    total_step * epsilon_ratio, each 'constant' or 'linear'.  Shared by `IQL` and the batched training driver."""
    lr_init = model_config.getfloat('lr_init')
    lr_decay = model_config.get('lr_decay')
    lr = Scheduler(lr_init, decay=lr_decay) if lr_decay == 'constant' else \
        Scheduler(lr_init, model_config.getfloat('lr_min'), total_step, decay=lr_decay)
    eps_init = model_config.getfloat('epsilon_init')
    eps_decay = model_config.get('epsilon_decay')
    eps = Scheduler(eps_init, decay=eps_decay) if eps_decay == 'constant' else \
        Scheduler(eps_init, model_config.getfloat('epsilon_min'), total_step * model_config.getfloat('epsilon_ratio'),
                  decay=eps_decay)
    return lr, eps


class IQL:
    """Independent Q-learning (agents/models.py:264-376, agents/policies.py:285-389): per-agent
    linear ('lr', LRQPolicy) or two-layer ('dqn', DeepQPolicy) Q network, epsilon-greedy exploration,
    1-step TD target WITHOUT a target network (policies.py:318-322), Adam, replay buffer, 10
    minibatches per agent per backward() (models.py:337-345).

    This is BASELINE config 1 ("reference plumbing", single env): it runs on PyTorch tensor ops
    (device tensors + torch.optim.Adam), not on hand-written kernels — it is not part of the measured
    hot path (DESIGN.md §7)."""
    name = 'iql'

    def __init__(self, n_s_ls, n_a_ls, n_w_ls, total_step, model_config, seed=0, model_type='dqn', device=None):
        from .utils import ReplayBuffer
        self.model_type = model_type
        self.n_agent = len(n_s_ls)
        self.reward_clip = model_config.getfloat('reward_clip')
        self.reward_norm = model_config.getfloat('reward_norm')
        self.n_s_ls, self.n_a_ls, self.n_w_ls = list(n_s_ls), list(n_a_ls), list(n_w_ls)
        self.n_step = model_config.getint('batch_size')
        self.sess = None
        self.total_step = total_step
        self.dev = torch.device(device if device is not None else ('cuda' if torch.cuda.is_available() else 'cpu'))
        self.gamma = model_config.getfloat('gamma')
        self.max_grad_norm = model_config.getfloat('max_grad_norm')
        rng = np.random.RandomState(seed)
        self._np_rng = np.random.RandomState(seed + 1)
        from .layout import ortho_init
        self.nets, self.opts = [], []
        for n_s, n_a, n_w in zip(self.n_s_ls, self.n_a_ls, self.n_w_ls):
            layers = {}
            if model_type == 'dqn':
                n_fc, n_h = model_config.getint('num_fc'), model_config.getint('num_h')
                if n_w == 0:
                    layers['q_fcw'] = (n_s, n_fc); width = n_fc
                else:
                    layers['q_fcw'] = (n_s - n_w, n_fc); layers['q_fct'] = (n_w, n_fc // 4); width = n_fc + n_fc // 4
                layers['q_fc_0'] = (width, n_h); layers['q'] = (n_h, n_a)
            else:
                layers['q'] = (n_s, n_a)
            params = {}
            for k, shp in layers.items():
                params[k + '/w'] = torch.tensor(ortho_init(rng, shp), device=self.dev, requires_grad=True)
                params[k + '/b'] = torch.zeros(shp[1], device=self.dev, requires_grad=True)
            self.nets.append(params)
        if total_step:
            self.lr_scheduler, self.eps_scheduler = iql_schedulers(model_config, total_step)
            buffer_size = model_config.getfloat('buffer_size')
            self.trans_buffer_ls = [ReplayBuffer(buffer_size, self.n_step) for _ in range(self.n_agent)]
            # TF1 AdamOptimizer state (agents/policies.py:327): first / second moments per tensor and the step count
            self.adam = [dict(t=0, m={k: torch.zeros_like(v) for k, v in p.items()},
                              v={k: torch.zeros_like(v) for k, v in p.items()}) for p in self.nets]

    def _q(self, i, S):
        p, n_w = self.nets[i], self.n_w_ls[i]
        if self.model_type != 'dqn':
            return S @ p['q/w'] + p['q/b']
        if n_w == 0:
            h = torch.relu(S @ p['q_fcw/w'] + p['q_fcw/b'])
        else:
            n_s = S.shape[1] - n_w
            h = torch.cat([torch.relu(S[:, :n_s] @ p['q_fcw/w'] + p['q_fcw/b']),
                           torch.relu(S[:, n_s:] @ p['q_fct/w'] + p['q_fct/b'])], 1)
        h = torch.relu(h @ p['q_fc_0/w'] + p['q_fc_0/b'])
        return h @ p['q/w'] + p['q/b']

    def forward(self, obs, mode='act', stochastic=False):
        if mode == 'explore':
            eps = self.eps_scheduler.get(1)
        action, qs_ls = [], []
        for i in range(self.n_agent):
            with torch.no_grad():
                qs = self._q(i, torch.as_tensor(np.asarray(obs[i], np.float32)[None], device=self.dev))[0].cpu().numpy()
            if mode == 'explore' and self._np_rng.random_sample() < eps:
                action.append(int(self._np_rng.randint(self.n_a_ls[i])))
            elif not stochastic:
                action.append(int(np.argmax(qs)))
            else:
                pq = qs / np.sum(qs)
                action.append(int(self._np_rng.choice(np.arange(len(pq)), p=pq)))
            qs_ls.append(qs)
        return action, qs_ls

    def add_transition(self, obs, actions, rewards, next_obs, done):
        rewards = np.asarray(rewards, np.float64)
        if self.reward_norm:
            rewards = rewards / self.reward_norm
        if self.reward_clip:
            rewards = np.clip(rewards, -self.reward_clip, self.reward_clip)
        for i in range(self.n_agent):
            self.trans_buffer_ls[i].add_transition(obs[i], actions[i], rewards[i], next_obs[i], done)

    def td_update(self, i, obs, acts, next_obs, dones, rs, cur_lr):
        """One minibatch update of agent i = QPolicy.prepare_loss + backward (agents/policies.py:307-338,362-377):
        loss = mean((q(s)[a] - stop_grad(done ? r : r + gamma max_a' q(s')[a']))^2), same network for both (no target
        net), tf.clip_by_global_norm (g * clip / max(norm, clip)), TF1 Adam (lr_t = lr sqrt(1-b2^t)/(1-b1^t),
        var -= lr_t m / (sqrt(v) + 1e-8)).  Returns (loss, grad_norm)."""
        p = self.nets[i]
        S = torch.as_tensor(np.asarray(obs, np.float32), device=self.dev)
        S1 = torch.as_tensor(np.asarray(next_obs, np.float32), device=self.dev)
        A = torch.as_tensor(np.asarray(acts).astype(np.int64), device=self.dev)
        R = torch.as_tensor(np.asarray(rs, np.float32), device=self.dev)
        D = torch.as_tensor(np.asarray(dones).astype(bool), device=self.dev)
        q0 = self._q(i, S).gather(1, A[:, None])[:, 0]
        with torch.no_grad():
            tq = torch.where(D, R, R + self.gamma * self._q(i, S1).max(1)[0])
        loss = ((q0 - tq) ** 2).mean()
        self.td_means = (q0.detach().mean(), tq.mean())         # the summaries' q and tq (agents/policies.py:335-336)
        keys = list(p.keys())
        grads = torch.autograd.grad(loss, [p[k] for k in keys])
        norm = torch.sqrt(sum((g * g).sum() for g in grads))
        if self.max_grad_norm > 0:
            scale = self.max_grad_norm / torch.clamp(norm, min=self.max_grad_norm)
            grads = [g * scale for g in grads]
        st = self.adam[i]
        st['t'] += 1
        b1, b2, eps = 0.9, 0.999, 1e-8
        lr_t = cur_lr * np.sqrt(1.0 - b2 ** st['t']) / (1.0 - b1 ** st['t'])
        with torch.no_grad():
            for k, g in zip(keys, grads):
                st['m'][k] += (g - st['m'][k]) * (1.0 - b1)
                st['v'][k] += (g * g - st['v'][k]) * (1.0 - b2)
                p[k] -= lr_t * st['m'][k] / (torch.sqrt(st['v'][k]) + eps)
        return float(loss.detach()), float(norm)

    def backward(self, summary_writer=None, global_step=None):
        """With a writer (add_scalar(tag, value, step)), agent 0's loss, mean q, mean tq and pre-clip gradient norm of
        round k go in at global_step + k (agents/policies.py:331-338, agents/models.py:337-345)."""
        cur_lr = self.lr_scheduler.get(self.n_step)
        if self.trans_buffer_ls[0].size < self.trans_buffer_ls[0].batch_size:
            return
        name = self._prefix(0)[:-len('_q/')]
        for i in range(self.n_agent):
            for k in range(10):                                   # agents/models.py:337-345
                obs, acts, next_obs, rs, dones = self.trans_buffer_ls[i].sample_transition()
                loss, norm = self.td_update(i, obs, acts, next_obs, dones, rs, cur_lr)
                if i == 0 and summary_writer is not None:
                    q, tq = (float(x) for x in self.td_means)
                    for tag, v in (('loss', loss), ('q', q), ('tq', tq), ('gradnorm', norm)):
                        summary_writer.add_scalar('train/%s_%s' % (name, tag), v, global_step + k)

    def reset(self):
        return

    def _prefix(self, i):
        return '%s_%da_q/' % ('dqn' if self.model_type == 'dqn' else 'lr', i)      # agents/policies.py:343,346,383,386

    def named_weights(self):
        return {self._prefix(i) + k: v.detach().cpu().numpy() for i, p in enumerate(self.nets) for k, v in p.items()}

    def load_named(self, named):
        for i, p in enumerate(self.nets):
            for k in p:
                arr = np.asarray(named[self._prefix(i) + k], np.float32)
                if tuple(arr.shape) != tuple(p[k].shape):
                    raise ValueError('tensor %r has shape %s, expected %s' % (self._prefix(i) + k, arr.shape, tuple(p[k].shape)))
                p[k].data.copy_(torch.from_numpy(arr))

    def save(self, model_dir, global_step):
        from . import checkpoint as ck
        ck.save_npz(os.path.join(model_dir, 'checkpoint-%d.npz' % int(global_step)), self.named_weights(),
                    {'step': np.int64(global_step)})

    def load(self, model_dir, checkpoint=None):
        from . import checkpoint as ck
        files = [f for f in os.listdir(model_dir)] if os.path.exists(model_dir) else []
        steps = [int(f.split('.')[0].split('-')[1]) for f in files
                 if f.startswith('checkpoint-') and len(f.split('.')[0].split('-')) == 2]
        if checkpoint is None and not steps:
            logging.error('Can not find old checkpoint for %s' % model_dir)
            return False
        step = int(checkpoint) if checkpoint is not None else max(steps)
        path = os.path.join(model_dir, 'checkpoint-%d.npz' % step)
        if not os.path.exists(path):
            logging.error('Can not find old checkpoint for %s' % model_dir)
            return False
        self.load_named(ck.load_npz(path)[0])
        return True
