"""Batched FC actor-critic learner: the reference's `FcACPolicy` (agents/policies.py:214-256; BASELINE config 2
"IA2C (FC policy)") for R replicas x A agents x 2 networks.

    h = concat(relu(fcw(wave)), relu(fct(wait)))  ->  relu(fc(h), 64)  ->  softmax head / value head

Same parameter vector layout as the LSTM learner with `PolicyLayout(recurrent=False)`: the LSTM block is replaced by
`wx` [dx, 64] + `bl` [64]; the ragged fc front end and the heads are unchanged, so the hand-written kernels of
csrc/tsc_learn.cu do the front end (tscl_fc_embed / tscl_fc_bwd_tc), the heads, sampling, loss and head gradients
(tscl_heads, tscl_heads_loss), returns and clip + RMSProp; the dense 160 x 64 layer in the middle runs on the
register-tiled fp32 kernels tscl_fc_hidden_fwd / tscl_fc_hidden_bwd (no library GEMM on this path).  There is no recurrent state: `done` is ignored by forward().
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from .. import _lib
from .. import dist as _dist
from .layout import PolicyLayout
from .learner import BatchedA2C, _p


class BatchedFcA2C(BatchedA2C):
    def __init__(self, layout: PolicyLayout, n_replicas: int, n_step: int, **kw):
        assert not layout.recurrent, "BatchedFcA2C needs PolicyLayout(recurrent=False)"
        kw["use_tc"] = False               # the fused tensor-core forward / BPTT kernels are LSTM-specific
        kw["store_acts"] = False
        super().__init__(layout, n_replicas, n_step, **kw)
        self.fc_bwd_tc = layout.fc_bwd_tc_ok      # front-end weight gradients on the tensor cores (fp32 inputs)

    # ------------------------------------------------------------------------------------------
    def forward(self, obs: torch.Tensor, done: bool = False, out_type: str = "pv", sample: bool = True):
        L, R, lib = self.lay, self.R, _lib.lib()
        commit = "p" in out_type
        want_act = sample and commit
        self._mm()
        _lib.check(lib.tscl_fc_embed(self._h, _p(self.P), _p(obs), C.c_int64(R), C.c_int64(R), C.c_int64(0),
                                     _p(self.X1), self._st()))
        _lib.check(lib.tscl_fc_hidden_fwd(self._h, _p(self.P), _p(self.X1), C.c_int64(R), _p(self.H1), self._st()))
        _lib.check(lib.tscl_heads(self._h, _p(self.P), _p(self.H1), C.c_int64(R), _p(self.pi), _p(self.val),
                                  _p(self.act) if want_act else None, C.c_uint64(self.seed),
                                  C.c_int64(self.n_forward), C.c_int64(self.replica0), self._st()))
        self.kernel_launches += 3
        if commit:
            self.n_forward += 1
        return self.pi, self.val, (self.act if want_act else None)

    # ------------------------------------------------------------------------------------------
    def backward(self, boot: Optional[torch.Tensor], lr: float, beta: float):
        assert self.t == self.T, "rollout buffer not full"
        L, R, T, U, A, lib = self.lay, self.R, self.T, self.lay.U, self.lay.A, _lib.lib()
        self._mm()
        st = self._st
        f32 = dict(dtype=torch.float32, device=self.dev)
        dpost = torch.tensor(self.done_post, **f32)
        if boot is None:
            self.boot.zero_()
        else:
            self.boot.copy_(boot)
        _lib.check(lib.tscl_returns(self._h, _p(self.rew_hist), _p(self.val_hist), _p(self.boot), _p(dpost),
                                    C.c_float(self.gamma), C.c_int32(T), C.c_int64(R), _p(self.Rs), _p(self.Adv), st()))
        self.G.zero_()
        self.stats.zero_()
        scale = _dist.grad_scale(T, 1, self.total_replicas)
        n_obs = L.n_obs
        for r0 in range(0, R, self.chunk):
            rc = min(self.chunk, R - r0)
            M = T * rc
            X = torch.empty(U, M, L.dx, **f32)
            H = torch.empty(U, M, L.h, **f32)
            dH = torch.empty(U, M, L.h, **f32)
            obs0 = self.obs_hist[0, r0:]
            _lib.check(lib.tscl_fc_embed(self._h, _p(self.P), _p(obs0), C.c_int64(M), C.c_int64(rc),
                                         C.c_int64(R * n_obs), _p(X), st()))
            _lib.check(lib.tscl_fc_hidden_fwd(self._h, _p(self.P), _p(X), C.c_int64(M), _p(H), st()))
            _lib.check(lib.tscl_heads_loss(self._h, _p(self.P), _p(H), _p(self.act_hist[0, r0:]), _p(self.Rs[0, r0:]),
                                           _p(self.Adv[0, r0:]), C.c_int64(M), C.c_int64(rc), C.c_int64(R * A),
                                           C.c_float(self.v_coef), C.c_float(beta), C.c_float(scale), None, _p(dH),
                                           _p(self.stats), None, _p(self.G), st()))
            dX = torch.empty(U, M, L.dx, **f32)
            # relu', dX = dH . W^T, dW += X^T dH, db += 1^T dH: own kernels (no library GEMM on this path)
            _lib.check(lib.tscl_fc_hidden_bwd(self._h, _p(self.P), _p(X), _p(H), _p(dH), C.c_int64(M), _p(dX), _p(self.G),
                                              st()))
            if self.fc_bwd_tc:
                _lib.check(lib.tscl_fc_bwd_tc(self._h, _p(obs0), _p(X), None, _p(dX), None, C.c_int64(M), C.c_int64(rc),
                                              C.c_int64(R * n_obs), _p(self.G), C.c_int32(0), st()))
            else:
                _lib.check(lib.tscl_fc_bwd(self._h, _p(obs0), _p(X), _p(dX), C.c_int64(M), C.c_int64(rc),
                                           C.c_int64(R * n_obs), _p(self.G), st()))
            self.kernel_launches += 6
        if self.pg is not None:
            _dist.allreduce_sum_(self.G, self.pg)
        _lib.check(lib.tscl_clip_rmsprop(self._h, _p(self.P), _p(self.G), _p(self.MS), _p(self.agent_of),
                                         C.c_float(self.max_grad_norm), C.c_float(lr), C.c_float(self.alpha),
                                         C.c_float(self.eps), _p(self.norms), st()))
        self.kernel_launches += 3
        self.obs_hist[0].copy_(self.obs_hist[T])
        self.last_done = bool(self.done_post[-1])
        self.t = 0
