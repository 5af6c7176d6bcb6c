"""`BatchedA2C`: all A per-intersection actor-critics, R replicas at once, on one GPU.

Device-side counterpart of reference agents/models.py (IA2C/MA2C) + agents/policies.py
(LstmACPolicy / FPLstmACPolicy) + agents/utils.py (OnPolicyBuffer).  Semantics kept:
  * two separate LSTM networks per agent, state zeroed inside the cell on a pre-decision done
    (agents/utils.py:104-105); 'v'-only forward does not advance the state (agents/policies.py:127-135);
  * BPTT over n_step from `states_bw`, refreshed from `states_fw` after each update (:153);
  * loss of agents/policies.py:41-52, per-agent clip_by_global_norm, TF1 RMSProp (:54-61);
  * n-step returns of OnPolicyBuffer (agents/utils.py:202-214), reward /= reward_norm then clip
    (agents/models.py:222-229).
Replicas share the weights: the gradient is the mean over replicas (and over ranks: one
`all_reduce(SUM)` of the flat gradient per update, then identical updates everywhere).

Population (`seeds` with K > 1 entries): K independent members of the same agent, member k with its own weights
(initialised from seeds[k]), RMSProp slot, gradient and packed images, on n_replicas replicas each; the rows
k*n_replicas .. (k+1)*n_replicas - 1 of every per-replica array are member k's.  One grouped forward launch
(tscl_policy_step_v2g) serves all members and samples member k with the key of its own one-member learner (seed
seeds[k], replica index relative to the member), so each member trains what `BatchedA2C(seed=seeds[k])` trains alone.
The update runs the one-member kernels chunk by chunk (a chunk never straddles two members) with the member's
pointers, then one clip + RMSProp and one repack per member.  `member(k)` is a solo-model view of member k.

Sweep (`hparams`, K dicts of SWEEP_KEYS next to `seeds`, which may then repeat): a population whose members also differ
in gamma, v_coef, max_grad_norm, RMSProp alpha / eps and reward_norm / reward_clip, and whose `backward` takes one lr
and one beta per member.  Each chunk's loss kernel takes its member's v_coef and beta, each member's clip + RMSProp its
own lr, max_grad_norm, alpha and eps; the returns (tscl_returns_g) and the device reward hand-over
(tscl_device_transition_g) read per-member device arrays when the members' values differ.

Shipping path (`use_tc`, the default): every kernel is hand-written — the fused wgmma forward
(csrc/tsc_policy_tc.cu: fc front end, gate GEMM, LSTM cell, heads, sampling, bf16 activation store), the wgmma
update (BPTT with TMA operand copies, dX = dZ.Wx^T, LSTM and fc weight gradients) and the SIMT kernels of
csrc/tsc_learn.cu (loss / head gradients, returns, clip + RMSProp).  No library GEMM runs on it.
`use_tc=False` selects the plain fp32 twin kernels (fc_embed, lstm_seq_fwd / bwd, heads, fc_bwd) that the reference
goldens pin at 2e-4; only on that path do the three plain batched products (X.Wx, dZ.Wx^T, [X|H]^T.dZ) go through
`torch.baddbmm / bmm` (fp32, TF32 only when `allow_tf32`).

Imitation (`teacher`, DESIGN §5 Imitation): A2C guided by a signal controller in DAgger form.  The student drives the
simulator; at every control step the trainer has the teacher label the state the student is in, into `teach_hist[t]`
(int32 [T][R][A], next to act_hist).  For every row (t, r) and agent i with pi the softmax over the agent's n_a_i
logits, a the sampled action, A the advantage, b the teacher's action and lam the update's imitation coefficient (one
float per update, one per member in a sweep), the loss gains  -lam * log clip(pi_b, 1e-10, 1), summed with the A2C
terms' scale = 1 / (n_step * R_total).  Its gradient at the logits is  scale * lam * (pi_j - [j == b])  when pi_b is not
clipped and 0 when it is: the policy-gradient term with A := lam and a := b, added in the same pass of the kernels that
compute the head gradients (tscl_lstm_seq_bwd_tc_heads_imit, tscl_heads_loss_imit).  The value head and the entropy
term do not change; at lam = 0 the update is plain A2C.  stats[3] receives agent 0's unweighted cross-entropy
sum -log clip(pi_b, 1e-10, 1) * scale.  Teachers (TEACHERS): 'maxpressure' (tsc_pressure_actions on the simulator's lane
counts) and 'greedy' (tsc_greedy_actions on obs_hist[t] with the training env's greedy program: the greedy rule on the
own-wave entries the student sees, normalised and clipped by the training config).  Without a teacher the learner
allocates and launches exactly what it does without the feature.
"""
from __future__ import annotations

import ctypes as C
import os
import types
from typing import Optional, Sequence

import numpy as np
import torch

from .. import _lib
from .. import dist as _dist
from .layout import PolicyLayout


_p = _lib.ptr


def check_population(seeds, seed, n_replicas, chunk, process_group):
    """The member seeds of a learner: [seed] without `seeds`, else the list, which must hold distinct seeds; with
    more than one member, n_replicas (per member) must be a multiple of 64 (a forward tile never straddles two
    members), the update chunk min(chunk, n_replicas) must divide it, and there is no process group."""
    if seeds is None:
        return [int(seed)]
    seeds = [int(s) for s in seeds]
    if not seeds:
        raise ValueError("a population needs at least one seed")
    if len(set(seeds)) != len(seeds):
        raise ValueError("population seeds must be distinct (got %s)" % seeds)
    return _check_members(seeds, n_replicas, chunk, process_group)


# controllers that can label a student's state with one action per agent (BatchedA2C(teacher=...)).  Fixed-time, tuned
# fixed-time and actuated control cannot: their program phases include yellow and all-red, a phase may change inside a
# control interval, so there is no action label to give.
TEACHERS = ("maxpressure", "greedy")
NO_LABEL_CONTROLLERS = ("fixedtime", "actuated")


def check_teacher(teacher):
    """`teacher` if it is None or one of TEACHERS, else ValueError naming it (and why, for the program controllers)."""
    if teacher is None or teacher in TEACHERS:
        return teacher
    if teacher in NO_LABEL_CONTROLLERS:
        raise ValueError("teacher %r cannot label states: its signal program's phases include yellow and all-red and "
                         "a phase can change inside a control interval, so there is no action to imitate (teachers: %s)"
                         % (teacher, ", ".join(TEACHERS)))
    raise ValueError("unknown teacher %r (teachers: %s)" % (teacher, ", ".join(TEACHERS)))


def check_imit(v, name="imitation coefficient"):
    """An imitation coefficient as a float: finite and >= 0, else ValueError."""
    v = float(v)
    if not np.isfinite(v) or v < 0:
        raise ValueError("the %s must be finite and >= 0 (got %r)" % (name, v))
    return v


# the learner values a sweep member sets for itself (BatchedA2C(hparams=...)); lr and beta come with each backward
SWEEP_KEYS = ("gamma", "v_coef", "max_grad_norm", "alpha", "eps", "reward_norm", "reward_clip")


def check_sweep(seeds, hparams, n_replicas, chunk, process_group):
    """(seeds, hparams) of a sweep learner: one seed per member (seeds may repeat) and one dict per member holding
    exactly SWEEP_KEYS (reward_norm / reward_clip None or 0: off), under check_population's rules for replicas, the update
    chunk and the process group."""
    if seeds is None:
        raise ValueError("a sweep takes `seeds`, one per member")
    seeds, hparams = [int(s) for s in seeds], [dict(h) for h in hparams]
    if len(seeds) != len(hparams):
        raise ValueError("a sweep takes one seed per member (got %d seeds for %d members)" % (len(seeds), len(hparams)))
    for k, h in enumerate(hparams):
        if set(h) != set(SWEEP_KEYS):
            raise ValueError("member %d's hyperparameters must be exactly %s (got %s)" % (k, SWEEP_KEYS, sorted(h)))
    _check_members(seeds, n_replicas, chunk, process_group)
    return seeds, [{key: float(h[key] or 0.0) for key in SWEEP_KEYS} for h in hparams]


def _check_members(seeds, n_replicas, chunk, process_group):
    if not seeds:
        raise ValueError("a population needs at least one seed")
    if any(s < 0 or s >= 1 << 63 for s in seeds):
        raise ValueError("population seeds must lie in [0, 2^63) (got %s)" % seeds)
    if len(seeds) > 1:
        R_m, rc = int(n_replicas), min(int(chunk), int(n_replicas))
        if R_m <= 0 or R_m % 64:
            raise ValueError("a population needs a multiple of 64 replicas per member (got %d)" % R_m)
        if R_m % rc:
            raise ValueError("the update chunk (%d) must divide the replicas per member (%d)" % (rc, R_m))
        if process_group is not None:
            raise ValueError("a population trains in one process: it takes no process group")
    return seeds


# fc widths dx of the fused v2 forward and of the fused dX / fc weight-gradient kernel (P2_DX_OK, csrc/tsc_policy_tc.cu):
# grid MA2C 224, Monaco MA2C 192, grid IA2C 160, Monaco IA2C 128 at the reference's num_fw 128 / num_ft 32 / num_fp 64
V2_DX = (128, 160, 192, 224)


def learner_paths(layout: PolicyLayout, use_tc: bool = True, K: int = 1, dx_library: bool = False):
    """The kernels `BatchedA2C(layout, use_tc=use_tc)` with K members runs, as a namespace:
      forward   'v2' (tscl_policy_step_v2: fused fc front end, LSTM and heads on the tensor cores, activation store),
                'v1' (tscl_policy_step: fc front end in fp32; wave blocks of at most 32 inputs) or 'fp32' (the twin kernels);
      update    with the activation store on: 'lean' (every update kernel reads the bf16 store, dX fused into the fc weight
                gradients), 'store' (the store unpacked to fp32, dX by a torch product, SIMT tscl_fc_bwd: the layout has no
                spare input slot for the bias column of the tensor-core fc kernels); 'recompute' (no store: the forward is
                recomputed in fp32 per chunk) or 'fp32' (use_tc off).  Without the store every 'lean' / 'store' layout
                recomputes too;
      and the flags BatchedA2C keeps: use_tc, tc_v2, dx_fusable, dx_own, dx_fc_fused, bwd_tc, fc_bwd_tc, wgrad_tc.
    `dx_library` (TSC_DX_LIBRARY=1) replaces the stand-alone dX kernel by the library GEMM.  Raises ValueError for a
    layout the tensor-core forward does not serve, and for a population (K > 1) without the fused forward and dX."""
    L = layout
    use_tc = bool(use_tc) and L.dx % 16 == 0 and L.kw > 0              # else: the fp32 kernels
    if use_tc and L.dx > 224:
        # the fused forwards keep [Wx;Wh] resident in shared memory: 224 + 64 input rows is the most that fits
        raise ValueError("the tensor-core policy forward supports dx <= 224 (got %d); use use_tc=False" % L.dx)
    tc_v2 = use_tc and L.dx in V2_DX
    if use_tc and not tc_v2 and L.kw != 32:
        # the v1 kernel stages a 32-wide wave block (tscl_policy_step)
        raise ValueError("no tensor-core policy forward for fc width dx = %d with a wave block of %d inputs: the fused "
                         "forward takes dx in %s, the v1 forward other multiples of 16 up to 224 with wave blocks of at "
                         "most 32 inputs; change num_fw or use use_tc=False" % (L.dx, int(L.n_wave.max()), V2_DX))
    if K > 1 and not tc_v2:
        raise ValueError("a population needs the fused tensor-core forward (use_tc with fc width %s; got use_tc=%s, dx=%d)"
                         % (", ".join(map(str, V2_DX)), use_tc, L.dx))
    dx_own = use_tc and L.dx <= 224 and not dx_library          # stand-alone dX = dZ . Wx^T kernel (tscl_dx_tc)
    p = types.SimpleNamespace(
        use_tc=use_tc, tc_v2=tc_v2,
        dx_fusable=use_tc and L.dx % 32 == 0 and L.dx <= 256,  # dX inside the BPTT kernel (BatchedA2C.dx_fused)
        dx_own=dx_own,
        # dX fused into the fc weight-gradient kernel (tscl_dx_fc_bwd_tc: dX never reaches memory) at the v2 widths
        dx_fc_fused=dx_own and tc_v2,
        bwd_tc=use_tc,
        fc_bwd_tc=use_tc and L.fc_bwd_tc_ok,                    # front-end weight gradients on the tensor cores
        wgrad_tc=use_tc and L.dx % 8 == 0 and L.dx <= 240)      # LSTM weight gradients on the tensor cores
    if K > 1 and not p.dx_fc_fused:
        raise ValueError("a population needs dX fused into the fc weight-gradient kernel (unset TSC_DX_LIBRARY)")
    p.forward = "v2" if tc_v2 else "v1" if use_tc else "fp32"
    p.update = ("fp32" if not use_tc else "recompute" if not tc_v2 else
                "lean" if p.fc_bwd_tc and p.wgrad_tc else "store")
    return p


def deterministic_refusal(paths, store_acts: bool) -> Optional[str]:
    """Why `BatchedA2C(deterministic=True)` with kernel paths `paths` (learner_paths) and activation store `store_acts`
    cannot run its update in a fixed summation order, or None: only the lean update (the BPTT with the heads inside,
    the all-bf16 LSTM weight gradients, dX fused into the fc weight gradients) has deterministic kernels."""
    if not paths.use_tc:
        return "use_tc=False selects the fp32 twin kernels, which add their gradients with atomics"
    if paths.update != "lean":
        return ("this layout's update is %r, not the lean tensor-core update (the only one with deterministic kernels)"
                % paths.update)
    if not paths.dx_fc_fused:
        return "TSC_DX_LIBRARY=1 replaces the fused dX / fc weight-gradient kernel, which has the deterministic form"
    if os.environ.get("TSC_BPTT_HEADS", "1") == "0":
        return "TSC_BPTT_HEADS=0 selects tscl_heads_loss, which has no deterministic form"
    if not store_acts:
        return "the update must back-propagate through the activation store (store_acts off or it does not fit)"
    return None


class BatchedA2C:
    def __init__(self, layout: PolicyLayout, n_replicas: int, n_step: int, gamma: float = 0.99,
                 v_coef: float = 0.5, max_grad_norm: float = 40.0, alpha: float = 0.99, eps: float = 1e-5,
                 reward_norm: float = 1.0, reward_clip: float = 0.0, seed: int = 0, device: int = 0,
                 chunk: int = 1024, replica0: int = 0, total_replicas: Optional[int] = None,
                 process_group=None, allow_tf32: bool = True, use_tc: bool = True,
                 store_acts: Optional[bool] = None, seeds: Optional[Sequence[int]] = None,
                 hparams: Optional[Sequence[dict]] = None, deterministic: bool = False,
                 teacher: Optional[str] = None):
        self.teacher = check_teacher(teacher)
        if deterministic:       # the layout / switch refusals, before any device work
            why = deterministic_refusal(learner_paths(layout, use_tc, 1 if seeds is None else len(seeds),
                                                      os.environ.get("TSC_DX_LIBRARY", "0") == "1"),
                                        store_acts is not False)
            if why:
                raise ValueError("deterministic=True needs the lean update: " + why)
        if hparams is None:
            self.seeds = check_population(seeds, seed, n_replicas, chunk, process_group)
            self.hp = [dict(gamma=gamma, v_coef=v_coef, max_grad_norm=max_grad_norm, alpha=alpha, eps=eps,
                            reward_norm=reward_norm, reward_clip=reward_clip)] * len(self.seeds)
        else:                                 # a sweep: member 0's values stand for the learner's scalars
            self.seeds, self.hp = check_sweep(seeds, hparams, n_replicas, chunk, process_group)
            gamma, v_coef, max_grad_norm, alpha, eps, reward_norm, reward_clip = (self.hp[0][k] for k in SWEEP_KEYS)
        seed = self.seeds[0]                  # with `seeds`, a one-member population is the solo learner of seeds[0]
        self.K, self.R_m = len(self.seeds), int(n_replicas)
        self.paths = learner_paths(layout, use_tc, self.K, os.environ.get("TSC_DX_LIBRARY", "0") == "1")
        if not torch.cuda.is_available():
            raise RuntimeError("BatchedA2C needs a CUDA device (no CPU fallback exists)")
        self.lay, self.R, self.T = layout, self.K * int(n_replicas), int(n_step)
        self.gamma, self.v_coef, self.max_grad_norm = gamma, v_coef, max_grad_norm
        self.alpha, self.eps = alpha, eps
        self.reward_norm, self.reward_clip = reward_norm, reward_clip
        self.seed, self.replica0 = int(seed), int(replica0)
        self.total_replicas = int(total_replicas or n_replicas)
        self.pg = process_group
        self.allow_tf32 = allow_tf32
        self.dev = torch.device("cuda", device)
        self.chunk = min(int(chunk), self.R_m if self.K > 1 else self.R)
        lib = _lib.lib()
        self._cd = layout.as_c()
        h = C.c_void_p()
        _lib.check(lib.tscl_create(C.byref(self._cd), device, C.byref(h)))
        self._h = h
        # deterministic: the update kernels add in a fixed order (tscl_set_deterministic; same bits run to run)
        self.deterministic = bool(deterministic)
        if self.deterministic:
            _lib.check(lib.tscl_set_deterministic(h, 1, 0))
        L, R, T, U, A = layout, self.R, self.T, layout.U, layout.A
        f32 = dict(dtype=torch.float32, device=self.dev)
        if self.K == 1:
            self.P = torch.from_numpy(layout.init_params(seed)).to(self.dev)
        else:                                                  # [K][n_params], member k from its own seed
            self.P = torch.from_numpy(np.stack([layout.init_params(s) for s in self.seeds])).to(self.dev)
        self.G = torch.zeros_like(self.P)
        self.MS = torch.ones_like(self.P)                      # TF1 RMSProp slot "rms" starts at 1
        self.agent_of = torch.from_numpy(layout.agent_of).to(self.dev)
        self.norms = torch.zeros(A, **f32) if self.K == 1 else torch.zeros(self.K, A, **f32)
        self.stats = torch.zeros(4, **f32) if self.K == 1 else torch.zeros(self.K, 4, **f32)
        # parameter views of the fp32 twin path (K = 1 only)
        self.pv, self.gv = (layout.views(self.P), layout.views(self.G)) if self.K == 1 else (None, None)
        # recurrent state: [U][R][h] each
        self.c_fw = torch.zeros(U, R, L.h, **f32); self.h_fw = torch.zeros(U, R, L.h, **f32)
        self.c_bw = torch.zeros_like(self.c_fw); self.h_bw = torch.zeros_like(self.h_fw)
        self.c_tmp = torch.zeros_like(self.c_fw); self.h_tmp = torch.zeros_like(self.h_fw)
        # per-step work buffers
        self.X1 = torch.empty(U, R, L.dx, **f32)
        self.Z1 = torch.empty(U, R, 4 * L.h, **f32)
        self.H1 = torch.empty(U, R, L.h, **f32)
        self.pi = torch.zeros(R, A, L.max_na, **f32)
        self.val = torch.zeros(R, A, **f32)
        self.act = torch.zeros(R, A, dtype=torch.int32, device=self.dev)
        self.boot = torch.zeros(R, A, **f32)
        # rollout storage; obs slot t is what forward consumed at step t, slot T is the next obs
        self.obs_hist = torch.zeros(T + 1, R, L.n_obs, **f32)
        self.act_hist = torch.zeros(T, R, A, dtype=torch.int32, device=self.dev)
        self.rew_hist = torch.zeros(T, R, A, **f32)
        self.val_hist = torch.zeros(T, R, A, **f32)
        self.Rs = torch.zeros(T, R, A, **f32); self.Adv = torch.zeros(T, R, A, **f32)
        # the teacher's action of every rollout row (written by the trainer before each simulator step)
        self.teach_hist = torch.zeros(T, R, A, dtype=torch.int32, device=self.dev) if self.teacher else None
        self.done_pre = [0.0] * T
        self.done_post = [0.0] * T
        self.last_done = False      # OnPolicyBuffer.reset(done) carries the last done (agents/utils.py:187-193)
        self.t = 0
        self.n_forward = 0
        self._one = torch.zeros(1, **f32)
        self._upd_bufs = None
        self.kernel_launches = 0
        # fused tensor-core forward (csrc/tsc_policy_tc.cu): bf16 image of [Wx;Wh], refreshed after every update; the fc
        # front end on the tensor cores too at the V2_DX widths, other widths take the v1 kernel (learner_paths)
        paths = self.paths
        self.use_tc, self.tc_v2 = paths.use_tc, paths.tc_v2
        mdim = () if self.K == 1 else (self.K,)                # packed images per member
        self.Wp = torch.zeros(*mdim, U, ((L.dx + L.h) // 8) * 4 * L.h * 8 + 8 * L.dx * 8, dtype=torch.bfloat16,
                              device=self.dev)
        self.Wt = torch.zeros(*mdim, U, 32, L.h, 8, dtype=torch.bfloat16, device=self.dev)    # Wh^T image for the BPTT MMA
        self.Wxt = torch.zeros(*mdim, U, 32, L.dx, 8, dtype=torch.bfloat16, device=self.dev)  # Wx^T image: dX fused into the BPTT
        self.seeds_dev = torch.tensor(self.seeds, dtype=torch.int64, device=self.dev) if self.K > 1 else None
        # a sweep's per-member device values, only where the members differ (else the one-member kernels run)
        differ = lambda *keys: any(len({h[k] for h in self.hp}) > 1 for k in keys)
        per = lambda key: torch.tensor([h[key] for h in self.hp], **f32)
        self.gamma_dev = per("gamma") if differ("gamma") else None
        self.rscale_differs = differ("reward_norm", "reward_clip")
        self.rnorm_dev, self.rclip_dev = (per("reward_norm"), per("reward_clip")) if self.rscale_differs else (None, None)
        # fusing dX into the BPTT step lengthens its serial per-step chain, so the default keeps dX as a separate
        # product; `dx_fused = True` selects the fused kernel (tests/test_update_bench_size_gpu.py: test_fused_dx_bptt,
        # test_whole_update_matches_chunked_reference)
        self.dx_fused = False
        self.dx_fusable = paths.dx_fusable
        # stand-alone dX = dZ . Wx^T kernel (tscl_dx_tc); False falls back to the library GEMM (A/B measurements only)
        self.dx_own = paths.dx_own
        # False runs tscl_dx_tc + tscl_fc_bwd_tc (tests/test_dx_fc_bwd_fused_gpu.py compares the two)
        self.dx_fc_fused = paths.dx_fc_fused
        self.bwd_tc, self.fc_bwd_tc, self.wgrad_tc = paths.bwd_tc, paths.fc_bwd_tc, paths.wgrad_tc
        self.fused_heads = True                                  # head weight gradients inside tscl_heads_loss
        # on the lean path the BPTT kernel computes the loss gradients at the heads itself (tscl_lstm_seq_bwd_tc_heads:
        # same dZ bits, no fp32 dH round trip) and, for one member, runs once over every chunk; TSC_BPTT_HEADS=0 restores
        # tscl_heads_loss + one tscl_lstm_seq_bwd_tc per chunk (A/B measurements)
        self.heads_in_bptt = os.environ.get("TSC_BPTT_HEADS", "1") != "0"
        self._dz_all = None
        self.pack_weights()
        # bf16 activation store of the rollout's own forward pass (written by the v2 kernel): the update then
        # back-propagates through it instead of recomputing fc + gate GEMM + LSTM forward.
        need = U * T * R * (L.dx + 4 * L.h + 2 * L.h) * 2
        if store_acts is None:
            free, _ = torch.cuda.mem_get_info(self.dev)
            store_acts = self.tc_v2 and need < 0.5 * free
        self.store_acts = bool(store_acts) and self.tc_v2 and (R % self.chunk == 0)
        if self.K > 1 and not self.store_acts:
            raise ValueError("a population back-propagates through the activation store, which does not fit: %.2f GB "
                             "for %d x %d replicas" % (need / 1e9, self.K, self.R_m))
        self.st_x = self.st_g = self.st_c = self.st_h = None
        if self.store_acts:       # [R/chunk][U][T][chunk][w]: every update chunk is one contiguous block
            bf = dict(dtype=torch.bfloat16, device=self.dev)
            nc, rc_ = R // self.chunk, self.chunk
            self.st_x = torch.zeros(nc, U, T, rc_, L.dx, **bf); self.st_g = torch.zeros(nc, U, T, rc_, 4 * L.h, **bf)
            self.st_c = torch.zeros(nc, U, T, rc_, L.h, **bf); self.st_h = torch.zeros(nc, U, T, rc_, L.h, **bf)
        self._acts_ok = [False] * T      # step t of the current rollout was produced by a storing forward()
        if self.deterministic and not self.store_acts:
            raise ValueError("deterministic=True needs the lean update: the update must back-propagate through the "
                             "activation store, which does not fit (%.2f GB)" % (need / 1e9))

    def close(self):
        if getattr(self, "_h", None) is not None:
            _lib.lib().tscl_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def member(self, k: int):
        """Member k as a solo learner reads: its parameters P, RMSProp slot MS, packed image Wp, loss terms stats and
        gradient norms norms (views into the stacked tensors, so they follow training), with the layout and handle, and
        its own SWEEP_KEYS values."""
        if self.K == 1:
            return self
        return types.SimpleNamespace(lay=self.lay, _h=self._h, dev=self.dev, use_tc=self.use_tc, tc_v2=self.tc_v2,
                                     paths=self.paths, K=1, P=self.P[k], MS=self.MS[k], Wp=self.Wp[k], stats=self.stats[k],
                                     norms=self.norms[k], seed=self.seeds[k], **self.hp[k])

    def _one_reward_scaling(self, what):
        if self.rscale_differs:
            raise ValueError("%s applies one reward_norm / reward_clip to every replica, but the sweep's members "
                             "differ in them; use the device-resident loop (add_transition_device)" % what)

    def _per_member(self, v, name):
        """lr / beta / imit of backward(): one value for every member, or a sequence of K"""
        if isinstance(v, (list, tuple, np.ndarray)):
            if len(v) != self.K:
                raise ValueError("%s takes one value per member (%d, got %d)" % (name, self.K, len(v)))
            return [float(x) for x in v]
        return [v] * self.K

    def _st(self):
        return _lib.stream(self.dev)

    def pack_weights(self):
        if self.K > 1:
            lib = _lib.lib()
            for k in range(self.K):
                _lib.check(lib.tscl_pack_weights(self._h, _p(self.P[k]), _p(self.Wp[k]), self._st()))
                _lib.check(lib.tscl_pack_wht(self._h, _p(self.P[k]), _p(self.Wt[k]), self._st()))
                _lib.check(lib.tscl_pack_wxt(self._h, _p(self.P[k]), _p(self.Wxt[k]), self._st()))
            self.kernel_launches += 3 * self.K
            return
        if self.use_tc:
            _lib.check(_lib.lib().tscl_pack_weights(self._h, _p(self.P), _p(self.Wp), self._st()))
            _lib.check(_lib.lib().tscl_pack_wht(self._h, _p(self.P), _p(self.Wt), self._st()))
            if self.dx_fusable or self.dx_own:
                _lib.check(_lib.lib().tscl_pack_wxt(self._h, _p(self.P), _p(self.Wxt), self._st()))
            self.wx_b = self.pv["wx"].to(torch.bfloat16)       # operand of the separate product dX = dZ . Wx^T
            self.kernel_launches += 3

    def _mm(self):
        # cuBLAS fp32 (or TF32 when allowed) for the plain batched GEMMs
        torch.backends.cuda.matmul.allow_tf32 = bool(self.allow_tf32)

    # ------------------------------------------------------------------------------------------
    def reset(self):
        """model.reset(): zero the LSTM states (agents/models.py:218-220, policies.py:120-123)."""
        for t in (self.c_fw, self.h_fw, self.c_bw, self.h_bw):
            t.zero_()

    def forward(self, obs: torch.Tensor, done: bool, out_type: str = "pv", sample: bool = True, to_hist: bool = False):
        """One decision for all replicas/agents.  obs [R, n_obs] device tensor.  Returns
        (pi [R, A, max_na], val [R, A], act [R, A] or None); 'v' does not advance the state.
        `to_hist` (fused tensor-core forward only): values / actions are written straight into the rollout slots
        val_hist[t] / act_hist[t] (what add_transition would copy there); those views are returned."""
        L, R, lib = self.lay, self.R, _lib.lib()
        commit = "p" in out_type
        want_act = sample and commit
        to_hist = to_hist and self.use_tc and self.tc_v2 and want_act and self.t < self.T
        val_o, act_o = (self.val_hist[self.t], self.act_hist[self.t]) if to_hist else (self.val, self.act)
        if self.K > 1:
            c1, h1 = (self.c_fw, self.h_fw) if commit else (self.c_tmp, self.h_tmp)
            store = commit and self.t < self.T
            st = (_p(self.st_x), _p(self.st_g), _p(self.st_c), _p(self.st_h)) if store else (None,) * 4
            _lib.check(lib.tscl_policy_step_v2g(
                self._h, _p(self.P), self.P.shape[1], _p(self.Wp), self.Wp[0].numel(), _p(obs), self.K, self.R_m,
                _p(self.c_fw), _p(self.h_fw), _p(c1), _p(h1), _p(self.pi), _p(val_o), _p(act_o) if want_act else None,
                1 if done else 0, _p(self.seeds_dev), self.n_forward, *st, self.t if store else 0, self.T, self.chunk,
                self._st()))
            if store:
                self._acts_ok[self.t] = True
            self.kernel_launches += 1
            if commit:
                self.n_forward += 1
            self._hist_direct = to_hist
            return self.pi, val_o, (act_o if want_act else None)
        if self.use_tc:
            c1, h1 = (self.c_fw, self.h_fw) if commit else (self.c_tmp, self.h_tmp)
            args = (self._h, _p(self.P), _p(self.Wp), _p(obs), R, _p(self.c_fw), _p(self.h_fw), _p(c1),
                    _p(h1), _p(self.pi), _p(val_o), _p(act_o) if want_act else None,
                    1 if done else 0, self.seed, self.n_forward, self.replica0, None)
            if self.tc_v2:
                store = self.store_acts and commit and self.t < self.T
                st = (_p(self.st_x), _p(self.st_g), _p(self.st_c), _p(self.st_h)) if store else (None,) * 4
                _lib.check(lib.tscl_policy_step_v2(*args, *st, self.t if store else 0, self.T, self.chunk, self._st()))
                if commit and self.t < self.T:
                    self._acts_ok[self.t] = store
            else:
                _lib.check(lib.tscl_policy_step(*args, 0, self._st()))
            self.kernel_launches += 1
            if commit:
                self.n_forward += 1
            self._hist_direct = to_hist
            return self.pi, val_o, (act_o if want_act else None)
        self._mm()
        dflag = self._one.fill_(1.0 if done else 0.0)
        _lib.check(lib.tscl_fc_embed(self._h, _p(self.P), _p(obs), R, R, 0, _p(self.X1), self._st()))
        torch.baddbmm(self.pv["bl"].unsqueeze(1), self.X1, self.pv["wx"], out=self.Z1)
        c1, h1 = (self.c_fw, self.h_fw) if commit else (self.c_tmp, self.h_tmp)
        _lib.check(lib.tscl_lstm_seq_fwd(self._h, _p(self.P), _p(self.Z1), None, _p(self.H1), None, _p(self.c_fw),
                                         _p(self.h_fw), _p(c1), _p(h1), _p(dflag), 1, R, R, 0, self._st()))
        _lib.check(lib.tscl_heads(self._h, _p(self.P), _p(self.H1), R, _p(self.pi), _p(self.val),
                                  _p(self.act) if want_act else None, self.seed, self.n_forward, self.replica0,
                                  self._st()))
        self.kernel_launches += 3
        if commit:
            self.n_forward += 1
        return self.pi, self.val, (self.act if want_act else None)

    def forward_range(self, r0: int, n: int, done: bool, t: int, n_forward: int, stream=None, to_hist: bool = False):
        """forward() for the replica range [r0, r0 + n) only, on the current stream, for rollout slot `t` and decision
        counter `n_forward` (the caller may run ranges one step apart): reads obs_slot(t)[r0:r0+n], advances that
        range's recurrent state and writes its slices of pi / val / act (and of the activation store).  Ranges are
        independent.  Tensor-core path only; bookkeeping of the step: end_forward_ranges().
        `stream`: raw CUDA stream handle (default: torch's current stream).  `to_hist`: actions / values go straight into
        the rollout slots act_hist[t] / val_hist[t] (what add_transition would copy there) and those views are returned."""
        assert self.use_tc and self.tc_v2, "forward_range needs the fused tensor-core forward"
        assert self.K == 1, "forward_range serves one-member learners"
        L, R, A = self.lay, self.R, self.lay.A
        store = self.store_acts and t < self.T
        st = (_p(self.st_x), _p(self.st_g), _p(self.st_c), _p(self.st_h)) if store else (None,) * 4
        off = lambda t_, per_row: t_.data_ptr() + r0 * per_row * t_.element_size()
        _lib.check(_lib.lib().tscl_policy_step_v2r(
            self._h, _p(self.P), _p(self.Wp), off(self.obs_hist[t], L.n_obs), n, off(self.c_fw, L.h),
            off(self.h_fw, L.h), off(self.c_fw, L.h), off(self.h_fw, L.h), off(self.pi, A * L.max_na),
            off(self.val_hist[t] if to_hist else self.val, A), off(self.act_hist[t] if to_hist else self.act, A),
            1 if done else 0, self.seed, n_forward, self.replica0 + r0, None, *st, t if store else 0, self.T,
            self.chunk, R, r0, self._st() if stream is None else stream))
        self.kernel_launches += 1
        if t < self.T:
            self._acts_ok[t] = store
        if to_hist:
            return self.pi[r0:r0 + n], self.val_hist[t, r0:r0 + n], self.act_hist[t, r0:r0 + n]
        return self.pi[r0:r0 + n], self.val[r0:r0 + n], self.act[r0:r0 + n]

    def end_forward_ranges(self):
        """One decision step has been issued for every range."""
        self.n_forward += 1

    def add_transition_range(self, r0: int, n: int, reward: torch.Tensor):
        """add_transition() data movement for one replica range (reward [n, A]); finish the step with
        end_transition_ranges(done_pre, done_post)."""
        self._one_reward_scaling("add_transition_range")
        t = self.t
        r = reward
        if self.reward_norm:
            r = r / self.reward_norm
        if self.reward_clip:
            r = torch.clamp(r, -self.reward_clip, self.reward_clip)
        self.rew_hist[t, r0:r0 + n].copy_(r)
        self.act_hist[t, r0:r0 + n].copy_(self.act[r0:r0 + n])
        self.val_hist[t, r0:r0 + n].copy_(self.val[r0:r0 + n])

    def end_transition_ranges(self, done_pre: bool, done_post: bool):
        t = self.t
        self.done_pre[t] = 1.0 if done_pre else 0.0
        self.done_post[t] = 1.0 if done_post else 0.0
        self.t += 1

    # ------------------------------------------------------------------------------------------
    def obs_slot(self, t: Optional[int] = None) -> torch.Tensor:
        return self.obs_hist[self.t if t is None else t]

    def add_transition(self, reward: torch.Tensor, done_pre: bool, done_post: bool,
                       act: Optional[torch.Tensor] = None, val: Optional[torch.Tensor] = None):
        """Record step t: obs must already be in obs_slot(t) (the env writes there); actions and
        values default to the ones of the last forward().  agents/models.py:222-229."""
        self._one_reward_scaling("add_transition")
        t = self.t
        r = reward
        if self.reward_norm:
            r = r / self.reward_norm
        if self.reward_clip:
            r = torch.clamp(r, -self.reward_clip, self.reward_clip)
        self.rew_hist[t].copy_(r)
        self.act_hist[t].copy_(self.act if act is None else act)
        self.val_hist[t].copy_(self.val if val is None else val)
        self.done_pre[t] = 1.0 if done_pre else 0.0
        self.done_post[t] = 1.0 if done_post else 0.0
        self.t += 1

    def add_transition_device(self, reward: torch.Tensor, greward: torch.Tensor, rew_acc: torch.Tensor, done_pre: bool,
                              done_post: bool):
        """add_transition() of the device-resident loop in ONE launch: normalised / clipped reward into the rollout slot
        and the episode sum of the global reward; actions / values are already in their slots when the last forward ran
        with to_hist=True (copied otherwise).  Same arithmetic as add_transition (r * (1 / norm), clamp).  A sweep whose
        members differ in reward_norm / reward_clip scales each member's rows with its own (tscl_device_transition_g)."""
        t = self.t
        if self.rscale_differs:
            _lib.check(_lib.lib().tscl_device_transition_g(
                self._h, _p(reward), _p(self.rew_hist[t]), reward.numel(), _p(self.rnorm_dev), _p(self.rclip_dev),
                self.K, _p(greward), _p(rew_acc), greward.numel(), self._st()))
        else:
            _lib.check(_lib.lib().tscl_device_transition(
                self._h, _p(reward), _p(self.rew_hist[t]), reward.numel(), self.reward_norm or 0.0,
                self.reward_clip or 0.0, _p(greward), _p(rew_acc), greward.numel(), self._st()))
        if not getattr(self, "_hist_direct", False):
            self.act_hist[t].copy_(self.act)
            self.val_hist[t].copy_(self.val)
        self.done_pre[t] = 1.0 if done_pre else 0.0
        self.done_post[t] = 1.0 if done_post else 0.0
        self.t += 1

    def _bufs(self, rc, lean=False, dxb=True, dh=True, dzb=True):
        """Work buffers of one update chunk.  `lean`: every consumer reads the bf16 activation store itself and dZ / dX
        travel as bf16 between the tensor-core kernels, so only dH (fp32), dZb and dXb (bf16) exist (dXb only with
        `dxb`: the fused dX / fc kernel never writes dX; dH only with `dh`: not when the BPTT computes it; dZb only with
        `dzb`: not when one BPTT launch writes every chunk's dZ); the fp32 set is allocated the first time a fallback
        path needs it."""
        L, T, U = self.lay, self.T, self.lay.U
        f32 = dict(dtype=torch.float32, device=self.dev)
        if self._upd_bufs is None or self._upd_bufs["rc"] < rc:
            self._upd_bufs = dict(rc=rc)
        b = self._upd_bufs
        M = T * b["rc"]
        if (dh or not lean) and "dH" not in b:
            b["dH"] = torch.empty(U, M, L.h, **f32)
        if lean and dzb and "dZb" not in b:
            b["dZb"] = torch.empty(U, M, 4 * L.h, dtype=torch.bfloat16, device=self.dev)
        if lean and dxb and "dXb" not in b:
            b["dXb"] = torch.empty(U, M, L.dx, dtype=torch.bfloat16, device=self.dev)
        if not lean and "X" not in b:
            b.update(ZG=torch.empty(U, M, 4 * L.h, **f32), dX=torch.empty(U, M, L.dx, **f32),
                     X=torch.empty(U, M, L.dx, **f32), C=torch.empty(U, M, L.h, **f32), H=torch.empty(U, M, L.h, **f32),
                     Hp=torch.empty(U, M, L.h, **f32), dlog=torch.empty(U, M, L.max_na, **f32))
        return b

    def _dz_all_buf(self):
        """bf16 dZ of every chunk [R/chunk][U][T * chunk][4h] (one BPTT launch per update), or None when it does not fit
        in half of the free device memory (the activation store's rule)."""
        if self._dz_all is None:
            L, nc = self.lay, self.R // self.chunk
            need = nc * L.U * self.T * self.chunk * 4 * L.h * 2
            free, _ = torch.cuda.mem_get_info(self.dev)
            if need >= 0.5 * free:
                return None
            if self._upd_bufs is not None:          # the per-chunk dZ buffer is not needed beside it
                self._upd_bufs.pop("dZb", None)
            self._dz_all = torch.empty(nc, L.U, self.T * self.chunk, 4 * L.h, dtype=torch.bfloat16, device=self.dev)
        return self._dz_all

    def _bwd_heads(self, P, G, Wt, stats, r0, n_chunks, v_coef, beta, scale, dpre, dZb, imit=0.0):
        """tscl_lstm_seq_bwd_tc_heads over `n_chunks` chunks of the store from replica r0: loss gradients at the heads and
        BPTT in one kernel, dZ (bf16) into dZb, head weight gradients into G, agent 0's loss sums into stats; with a
        teacher the _imit form, toward teach_hist with coefficient `imit`."""
        ci, R, A = r0 // self.chunk, self.R, self.lay.A
        args = (self._h, _p(Wt), _p(P), _p(self.st_g[ci]), _p(self.st_c[ci]), _p(self.st_h[ci]), _p(self.c_bw), _p(dpre),
                _p(self.act_hist[0, r0:]), _p(self.Rs[0, r0:]), _p(self.Adv[0, r0:]), self.T, self.chunk, n_chunks, R, r0,
                R * A, v_coef, beta, scale, _p(dZb), _p(stats), _p(G))
        if self.teacher:
            _lib.check(_lib.lib().tscl_lstm_seq_bwd_tc_heads_imit(*args, _p(self.teach_hist[0, r0:]), imit, self._st()))
        else:
            _lib.check(_lib.lib().tscl_lstm_seq_bwd_tc_heads(*args, self._st()))

    def _imits(self, imit):
        """The update's imitation coefficient per member: with a teacher, `imit` (one value or one per member, each
        finite and >= 0); without one, `imit` must be 0."""
        imits = [check_imit(v) for v in self._per_member(imit, "imit")]
        if not self.teacher and any(imits):
            raise ValueError("an imitation coefficient (%s) needs a teacher (BatchedA2C(teacher=...))" % imits)
        return imits

    def backward(self, boot: Optional[torch.Tensor], lr: float, beta: float, imit=0.0):
        """One A2C update from the stored n_step rollout (agents/models.py:174-183).  `boot` is the
        bootstrap value [R, A] (None / zeros when the episode ended, utils.py:186-190).  `lr` / `beta`: one value, or one
        per member (a sweep's schedules).  `imit`: the imitation coefficient lam of a learner with a teacher, likewise
        (module docstring); 0 without one."""
        assert self.t == self.T, "rollout buffer not full"
        L, R, T, U, A, lib = self.lay, self.R, self.T, self.lay.U, self.lay.A, _lib.lib()
        lrs, betas = self._per_member(lr, "lr"), self._per_member(beta, "beta")
        imits = self._imits(imit)
        self._mm()
        st = self._st
        f32 = dict(dtype=torch.float32, device=self.dev)
        dpre = torch.tensor(self.done_pre, **f32)
        dpost = torch.tensor(self.done_post, **f32)
        if boot is None:
            self.boot.zero_()
        else:
            self.boot.copy_(boot)
        if self.gamma_dev is not None:
            _lib.check(lib.tscl_returns_g(self._h, _p(self.rew_hist), _p(self.val_hist), _p(self.boot), _p(dpost),
                                          _p(self.gamma_dev), self.K, T, R, _p(self.Rs), _p(self.Adv), st()))
        else:
            _lib.check(lib.tscl_returns(self._h, _p(self.rew_hist), _p(self.val_hist), _p(self.boot), _p(dpost),
                                        self.gamma, T, R, _p(self.Rs), _p(self.Adv), st()))
        self.G.zero_()
        self.stats.zero_()
        scale = _dist.grad_scale(T, 1, self.total_replicas)       # local SUM x 1/(n_step * R_total); ranks add up
        use_store = self.store_acts and all(self._acts_ok)
        if self.K > 1 and not use_store:
            raise RuntimeError("a population update needs every step of the rollout in the activation store")
        if self.deterministic:
            if not use_store:
                raise RuntimeError("a deterministic update needs every step of the rollout in the activation store "
                                   "(a step was not produced by a storing forward)")
            if self.dx_fused:
                raise ValueError("deterministic=True needs the lean update: dx_fused = True selects the BPTT kernel "
                                 "with dX inside, which has no deterministic form")
        n_obs = L.n_obs
        P, G, Wt, Wxt, stats = self.P, self.G, self.Wt, self.Wxt, self.stats
        k = 0
        lean = use_store and self.bwd_tc and self.fc_bwd_tc and self.wgrad_tc and self.fused_heads
        heads_bptt = lean and self.heads_in_bptt and not (self.dx_fused and self.dx_fusable)
        # one BPTT launch over every chunk (one member, and the all-chunk dZ fits); else one per chunk, the same bits
        dz_all = self._dz_all_buf() if heads_bptt and self.K == 1 and R > self.chunk else None
        if dz_all is not None:
            self._bwd_heads(P, G, Wt, stats, 0, R // self.chunk, self.hp[0]["v_coef"], betas[0], scale, dpre, dz_all,
                            imits[0])
            self.kernel_launches += 1
        for r0 in range(0, R, self.chunk):
            if self.K > 1:        # the member of this chunk: its weights, images, gradient and loss terms
                k = r0 // self.R_m
                P, G, Wt, Wxt, stats = self.P[k], self.G[k], self.Wt[k], self.Wxt[k], self.stats[k]
            rc = min(self.chunk, R - r0)
            M = T * rc
            ci = r0 // self.chunk
            all_tc = lean
            fuse_dx = all_tc and self.dx_fused and self.dx_fusable   # dX = dZ . Wx^T inside the BPTT kernel (second MMA per step)
            fuse_fc = all_tc and not fuse_dx and self.dx_fc_fused    # dX inside the fc weight-gradient kernel, never stored
            b = self._bufs(rc, lean=all_tc, dxb=not fuse_fc, dh=not heads_bptt, dzb=dz_all is None)
            X = Cc = H = Hp = dlog = ZG = dX = dZb = dXb = dH = None
            bf16 = dict(dtype=torch.bfloat16, device=self.dev)
            if b["rc"] == rc:
                dH = b.get("dH")
                if all_tc:
                    dZb, dXb = (b["dZb"] if dz_all is None else dz_all[ci]), b.get("dXb")
                else:
                    ZG, dX, X, Cc, H, Hp, dlog = (b[k] for k in ("ZG", "dX", "X", "C", "H", "Hp", "dlog"))
            else:               # tail chunk: dense temporaries of the right shape
                dH = torch.empty(U, M, L.h, **f32)
                if all_tc:
                    dZb = torch.empty(U, M, 4 * L.h, **bf16)
                    dXb = None if fuse_fc else torch.empty(U, M, L.dx, **bf16)
                else:
                    ZG, dX, X, Cc, H, Hp, dlog = (torch.empty(U, M, s_, **f32) for s_ in
                                                  (4 * L.h, L.dx, L.dx, L.h, L.h, L.h, L.max_na))
            obs0 = self.obs_hist[0, r0:]
            if all_tc:
                pass        # every consumer reads the bf16 activation store itself
            elif use_store:
                # activations of the rollout's forward pass (bf16 store -> fp32 chunk buffers)
                direct = self.bwd_tc        # the tensor-core BPTT kernel reads gates / c from the store itself
                _lib.check(lib.tscl_unpack_store(self._h, _p(self.st_x[ci]), _p(self.st_g[ci]), _p(self.st_c[ci]),
                                                 _p(self.st_h[ci]), _p(X), None if direct else _p(ZG),
                                                 None if direct else _p(Cc), _p(H), _p(Hp), _p(self.h_bw), _p(dpre), T,
                                                 rc, R, r0, st()))
            else:
                _lib.check(lib.tscl_fc_embed(self._h, _p(P), _p(obs0), M, rc, R * n_obs, _p(X), st()))
                torch.baddbmm(self.pv["bl"].unsqueeze(1), X, self.pv["wx"], out=ZG)
                _lib.check(lib.tscl_lstm_seq_fwd(self._h, _p(P), _p(ZG), _p(Cc), _p(H), _p(Hp), _p(self.c_bw),
                                                 _p(self.h_bw), None, None, _p(dpre), T, rc, R, r0, st()))
            hb = _p(self.st_h[ci]) if use_store else None
            if heads_bptt:      # heads + BPTT in one kernel (already run for every chunk when dz_all is set)
                if dz_all is None:
                    self._bwd_heads(P, G, Wt, stats, r0, 1, self.hp[k]["v_coef"], betas[k], scale, dpre, dZb, imits[k])
                    self.kernel_launches += 1
            else:
                args = (self._h, _p(P), None if all_tc else _p(H), _p(self.act_hist[0, r0:]), _p(self.Rs[0, r0:]),
                        _p(self.Adv[0, r0:]), M, rc, R * A, self.hp[k]["v_coef"], betas[k], scale,
                        None if self.fused_heads else _p(dlog), _p(dH), _p(stats), hb if all_tc else None,
                        _p(G) if self.fused_heads else None)
                if self.teacher:
                    _lib.check(lib.tscl_heads_loss_imit(*args, _p(self.teach_hist[0, r0:]), imits[k], st()))
                else:
                    _lib.check(lib.tscl_heads_loss(*args, st()))
                self.kernel_launches += 2
            if not self.fused_heads:
                # head weight / bias gradients (plain batched GEMM + column sums)
                self.gv["wo"].baddbmm_(H.transpose(1, 2), dlog)
                self.gv["bo"].add_(dlog.sum(dim=1))
            if heads_bptt:
                pass
            elif self.bwd_tc:
                gb = (_p(self.st_g[ci]), _p(self.st_c[ci])) if use_store else (None, None)
                _lib.check(lib.tscl_lstm_seq_bwd_tc_dx(self._h, _p(Wt), _p(ZG), _p(Cc), _p(dH), _p(self.c_bw), _p(dpre),
                                                       T, rc, R, r0, *gb, _p(dZb), _p(Wxt) if fuse_dx else None,
                                                       _p(dXb) if fuse_dx else None, st()))
            else:
                _lib.check(lib.tscl_lstm_seq_bwd(self._h, _p(P), _p(ZG), _p(Cc), _p(dH), _p(self.c_bw), _p(dpre), T, rc,
                                                 R, r0, st()))
            dZ = ZG
            if self.wgrad_tc:
                if use_store:
                    _lib.check(lib.tscl_wgrad_tc(self._h, _p(dZ), _p(dZb), None, _p(self.st_x[ci]), None,
                                                 _p(self.st_h[ci]), _p(self.h_bw), _p(dpre), T, rc, R, r0, _p(G), 0,
                                                 st()))
                else:
                    _lib.check(lib.tscl_wgrad_tc(self._h, _p(dZ), None, _p(X), None, _p(Hp), None, None, None, T, rc, R,
                                                 r0, _p(G), 0, st()))
            else:
                self.gv["wx"].baddbmm_(X.transpose(1, 2), dZ)
                self.gv["wh"].baddbmm_(Hp.transpose(1, 2), dZ)
                self.gv["bl"].add_(dZ.sum(dim=1))
            # dX = dZ . Wx^T: fused into the fc weight gradients on the shipping path (tscl_dx_fc_bwd_tc); else its own
            # warp-specialised wgmma kernel (tscl_dx_tc); a library GEMM only on the fp32 twin path, for dx > 224 and
            # under TSC_DX_LIBRARY=1 (A/B measurements)
            if fuse_fc:
                _lib.check(lib.tscl_dx_fc_bwd_tc(self._h, _p(obs0), _p(self.st_x[ci]), _p(dZb), _p(Wxt), M, rc,
                                                 R * n_obs, _p(G), st()))
            elif all_tc and not fuse_dx and self.dx_own:
                _lib.check(lib.tscl_dx_tc(self._h, _p(dZb), _p(Wxt), _p(dXb), M, st()))
            elif all_tc and not fuse_dx:
                torch.bmm(dZb, self.wx_b.transpose(1, 2), out=dXb)
            elif not all_tc:        # Wx of this chunk's member (self.pv is the K = 1 view only)
                torch.bmm(dZ, P[L.off_wx:L.off_wh].view(U, L.dx, 4 * L.h).transpose(1, 2), out=dX)
            if fuse_fc:
                pass            # the fc weight gradients came out of tscl_dx_fc_bwd_tc above
            elif self.fc_bwd_tc:
                xb = _p(self.st_x[ci]) if use_store else None
                _lib.check(lib.tscl_fc_bwd_tc(self._h, _p(obs0), None if all_tc else _p(X), xb, _p(dX), _p(dXb), M, rc,
                                              R * n_obs, _p(G), 0, st()))
            else:
                _lib.check(lib.tscl_fc_bwd(self._h, _p(obs0), _p(X), _p(dX), M, rc, R * n_obs, _p(G), st()))
            self.kernel_launches += 1 if fuse_fc else 2 if use_store else 3     # heads / BPTT counted above
        if self.pg is not None:
            _dist.allreduce_sum_(self.G, self.pg)
        for k in range(self.K):
            m = (lambda t_: t_) if self.K == 1 else (lambda t_: t_[k])
            hk = self.hp[k]
            _lib.check(lib.tscl_clip_rmsprop(self._h, _p(m(self.P)), _p(m(self.G)), _p(m(self.MS)), _p(self.agent_of),
                                             hk["max_grad_norm"], lrs[k], hk["alpha"], hk["eps"], _p(m(self.norms)),
                                             st()))
            self.kernel_launches += 3
        self.pack_weights()
        # states_bw <- states_fw (agents/policies.py:153); next rollout starts at slot 0
        self.c_bw.copy_(self.c_fw); self.h_bw.copy_(self.h_fw)
        self.obs_hist[0].copy_(self.obs_hist[T])
        self.last_done = bool(self.done_post[-1])
        self.t = 0
        self._acts_ok = [False] * T
