"""Flat parameter layout of the 2A per-intersection networks (pi and V per agent).

Mirrors the variable set of the reference graphs (agents/policies.py:87-96,202-209;
agents/utils.py:66-74,88-100): per unit u = 2*agent + net
    fcw {w [n_wave, fw], b}, fcf {w [n_fp, ff], b} (MA2C only), fct {w [n_wait, ft], b},
    lstm {wx [dx, 4h], wh [h, 4h], b [4h]}, head {w [h, n_out], b}   (n_out = n_a or 1).
The flat vector groups uniform kinds first so they are dense batched tensors
(wx [2A, dx, 4h], wh [2A, h, 4h], bl, wo [2A, h, max_na], bo), then the ragged fc layers.
`agent_of[i]` maps every float to its agent for the per-agent global-norm clip
(agents/policies.py:54-57).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence

import numpy as np


class CDims(C.Structure):
    _fields_ = [("n_agents", C.c_int32), ("n_obs", C.c_int32), ("max_na", C.c_int32),
                ("fw", C.c_int32), ("ff", C.c_int32), ("ft", C.c_int32), ("h", C.c_int32), ("dx", C.c_int32),
                ("obs_off", C.POINTER(C.c_int32)), ("n_wave", C.POINTER(C.c_int32)),
                ("n_wait", C.POINTER(C.c_int32)), ("n_fp", C.POINTER(C.c_int32)), ("n_a", C.POINTER(C.c_int32)),
                ("off_fcw_w", C.POINTER(C.c_int64)), ("off_fcw_b", C.POINTER(C.c_int64)),
                ("off_fcf_w", C.POINTER(C.c_int64)), ("off_fcf_b", C.POINTER(C.c_int64)),
                ("off_fct_w", C.POINTER(C.c_int64)), ("off_fct_b", C.POINTER(C.c_int64)),
                ("off_wx", C.c_int64), ("off_wh", C.c_int64), ("off_bl", C.c_int64),
                ("off_wo", C.c_int64), ("off_bo", C.c_int64), ("n_params", C.c_int64)]


class CQDims(C.Structure):
    _fields_ = [("n_agents", C.c_int32), ("n_obs", C.c_int32), ("max_na", C.c_int32), ("model", C.c_int32),
                ("n_fc", C.c_int32), ("n_ft", C.c_int32), ("n_h", C.c_int32),
                ("obs_off", C.POINTER(C.c_int32)), ("n_s", C.POINTER(C.c_int32)), ("n_w", C.POINTER(C.c_int32)),
                ("n_a", C.POINTER(C.c_int32)),
                ("off_fcw_w", C.POINTER(C.c_int64)), ("off_fcw_b", C.POINTER(C.c_int64)),
                ("off_fct_w", C.POINTER(C.c_int64)), ("off_fct_b", C.POINTER(C.c_int64)),
                ("off_fc0_w", C.POINTER(C.c_int64)), ("off_fc0_b", C.POINTER(C.c_int64)),
                ("off_q_w", C.POINTER(C.c_int64)), ("off_q_b", C.POINTER(C.c_int64)), ("n_params", C.c_int64)]


def ortho_init(rng: np.random.RandomState, shape, scale=np.sqrt(2)):
    """agents/utils.py:11-24 (lasagne-style orthogonal init via SVD)."""
    a = rng.standard_normal(shape)
    u, _, v = np.linalg.svd(a, full_matrices=False)
    q = u if u.shape == tuple(shape) else v
    return (scale * q.reshape(shape)).astype(np.float32)


class PolicyLayout:
    def __init__(self, n_s_ls: Sequence[int], n_a_ls: Sequence[int], n_w_ls: Sequence[int],
                 n_f_ls: Sequence[int], obs_off: Sequence[int], n_obs: int, fw: int, ft: int, ff: int = 0,
                 h: int = 64, max_na: int | None = None, recurrent: bool = True):
        """recurrent=False: FcACPolicy (agents/policies.py:214-256) — the LSTM block is replaced by one fc layer
        `wx` [dx, h] + `bl` [h] (relu), `wh` is empty."""
        self.recurrent = bool(recurrent)
        self.A = len(n_s_ls)
        if self.A > 255:
            raise ValueError("agent_of is a uint8 map (per-agent gradient-norm groups): at most 255 agents, got %d" % self.A)
        self.U = 2 * self.A
        self.n_a = np.asarray(n_a_ls, np.int32)
        self.n_wait = np.asarray(n_w_ls, np.int32)
        self.n_fp = np.asarray(n_f_ls, np.int32) if ff > 0 else np.zeros(self.A, np.int32)
        self.n_wave = (np.asarray(n_s_ls, np.int32) - self.n_wait - np.asarray(n_f_ls, np.int32)).astype(np.int32)
        self.obs_off = np.asarray(obs_off, np.int32)[:self.A].copy()
        self.n_obs, self.fw, self.ff, self.ft, self.h = int(n_obs), int(fw), int(ff), int(ft), int(h)
        if (self.n_wait == 0).all():
            self.ft = 0                                   # agents/policies.py:107-108 (n_w == 0)
        self.dx = self.fw + self.ff + self.ft
        # 64-slot input tile of the tensor-core kernels: wave block 32 or 48 wide, then 16 fingerprint slots
        # (+ 16 wait slots when the wave block is 32); one spare wave slot carries the bias column of tscl_fc_bwd_tc
        mw = int(self.n_wave.max())
        self.kw = 32 if mw <= 32 else (48 if (mw <= 48 and self.ft == 0) else 0)
        self.fc_bwd_tc_ok = self.kw > 0 and mw < self.kw and self.dx % 8 == 0 and self.dx <= 256
        self.max_na = int(max_na or self.n_a.max())
        U, dx, g4 = self.U, self.dx, (4 if self.recurrent else 1) * self.h
        hr = self.h if self.recurrent else 0              # rows of wh
        self.g4, self.hr = g4, hr
        off = 0
        self.off_wx = off; off += U * dx * g4
        self.off_wh = off; off += U * hr * g4
        self.off_bl = off; off += U * g4
        self.off_wo = off; off += U * self.h * self.max_na
        self.off_bo = off; off += U * self.max_na
        self.off_fcw_w = np.zeros(U, np.int64); self.off_fcw_b = np.zeros(U, np.int64)
        self.off_fcf_w = np.zeros(U, np.int64); self.off_fcf_b = np.zeros(U, np.int64)
        self.off_fct_w = np.zeros(U, np.int64); self.off_fct_b = np.zeros(U, np.int64)
        for u in range(U):
            a = u // 2
            self.off_fcw_w[u] = off; off += int(self.n_wave[a]) * self.fw
            self.off_fcw_b[u] = off; off += self.fw
            self.off_fcf_w[u] = off; off += int(self.n_fp[a]) * self.ff
            self.off_fcf_b[u] = off; off += self.ff
            self.off_fct_w[u] = off; off += int(self.n_wait[a]) * self.ft
            self.off_fct_b[u] = off; off += self.ft
        self.n_params = off
        # float -> agent map
        ag = np.zeros(off, np.uint8)
        unit_agent = np.repeat(np.arange(self.A, dtype=np.uint8), 2)
        ag[self.off_wx:self.off_wh] = np.repeat(unit_agent, dx * g4)
        ag[self.off_wh:self.off_bl] = np.repeat(unit_agent, hr * g4)
        ag[self.off_bl:self.off_wo] = np.repeat(unit_agent, g4)
        ag[self.off_wo:self.off_bo] = np.repeat(unit_agent, self.h * self.max_na)
        ag[self.off_bo:int(self.off_fcw_w[0])] = np.repeat(unit_agent, self.max_na)
        for u in range(U):
            end = int(self.off_fcw_w[u + 1]) if u + 1 < U else off
            ag[int(self.off_fcw_w[u]):end] = u // 2
        self.agent_of = ag

    # ---------------------------------------------------------------------------------------
    def as_c(self) -> CDims:
        c = CDims()
        c.n_agents, c.n_obs, c.max_na = self.A, self.n_obs, self.max_na
        c.fw, c.ff, c.ft, c.h, c.dx = self.fw, self.ff, self.ft, self.h, self.dx
        for name in ("obs_off", "n_wave", "n_wait", "n_fp", "n_a"):
            setattr(c, name, getattr(self, name).ctypes.data_as(C.POINTER(C.c_int32)))
        for name in ("off_fcw_w", "off_fcw_b", "off_fcf_w", "off_fcf_b", "off_fct_w", "off_fct_b"):
            setattr(c, name, getattr(self, name).ctypes.data_as(C.POINTER(C.c_int64)))
        c.off_wx, c.off_wh, c.off_bl, c.off_wo, c.off_bo = self.off_wx, self.off_wh, self.off_bl, self.off_wo, self.off_bo
        c.n_params = self.n_params
        c._keep = self
        return c

    def views(self, flat):
        """Named views into a flat numpy array or torch tensor."""
        U, dx, g4, h, mna = self.U, self.dx, self.g4, self.h, self.max_na
        v = {"wx": flat[self.off_wx:self.off_wh].reshape(U, dx, g4),
             "wh": flat[self.off_wh:self.off_bl].reshape(U, self.hr, g4),
             "bl": flat[self.off_bl:self.off_wo].reshape(U, g4),
             "wo": flat[self.off_wo:self.off_bo].reshape(U, h, mna),
             "bo": flat[self.off_bo:int(self.off_fcw_w[0])].reshape(U, mna)}
        for u in range(U):
            a = u // 2
            o = self
            v["fcw_w%d" % u] = flat[int(o.off_fcw_w[u]):int(o.off_fcw_b[u])].reshape(int(o.n_wave[a]), o.fw)
            v["fcw_b%d" % u] = flat[int(o.off_fcw_b[u]):int(o.off_fcf_w[u])]
            v["fcf_w%d" % u] = flat[int(o.off_fcf_w[u]):int(o.off_fcf_b[u])].reshape(int(o.n_fp[a]), o.ff)
            v["fcf_b%d" % u] = flat[int(o.off_fcf_b[u]):int(o.off_fct_w[u])]
            v["fct_w%d" % u] = flat[int(o.off_fct_w[u]):int(o.off_fct_b[u])].reshape(int(o.n_wait[a]), o.ft)
            v["fct_b%d" % u] = flat[int(o.off_fct_b[u]):int(o.off_fct_b[u]) + o.ft]
        return v

    def init_params(self, seed: int = 0) -> np.ndarray:
        """Orthogonal init, scale sqrt(2), zero biases (agents/utils.py:8,66-72,95-100), drawn in
        graph-construction order: per agent, pi net then V net (agents/policies.py:87-96)."""
        rng = np.random.RandomState(seed)
        flat = np.zeros(self.n_params, np.float32)
        v = self.views(flat)
        for u in range(self.U):
            a = u // 2
            v["fcw_w%d" % u][...] = ortho_init(rng, (int(self.n_wave[a]), self.fw))
            if self.ff > 0 and self.n_fp[a] > 0:
                v["fcf_w%d" % u][...] = ortho_init(rng, (int(self.n_fp[a]), self.ff))
            if self.ft > 0 and self.n_wait[a] > 0:
                v["fct_w%d" % u][...] = ortho_init(rng, (int(self.n_wait[a]), self.ft))
            v["wx"][u] = ortho_init(rng, (self.dx, self.g4))
            if self.recurrent:
                v["wh"][u] = ortho_init(rng, (self.h, 4 * self.h))
            n_out = int(self.n_a[a]) if u % 2 == 0 else 1
            v["wo"][u][:, :n_out] = ortho_init(rng, (self.h, n_out))
        return flat


class QLayout:
    """Flat fp32 parameter vector of the IQL Q networks (agents/policies.py:341-389), agent after agent, each agent's
    tensors in the order q_fcw/w, q_fcw/b, q_fct/w, q_fct/b, q_fc_0/w, q_fc_0/b, q/w, q/b (dqn; q_fct only for n_w > 0)
    or q/w, q/b (lr), every weight row-major [in][out] as `IQL.nets` holds it.  This is the `tscl_qdims` image the
    test-mode Q kernel reads (include/tsc_learn.h)."""
    OFF = {"q_fcw/w": "off_fcw_w", "q_fcw/b": "off_fcw_b", "q_fct/w": "off_fct_w", "q_fct/b": "off_fct_b",
           "q_fc_0/w": "off_fc0_w", "q_fc_0/b": "off_fc0_b", "q/w": "off_q_w", "q/b": "off_q_b"}

    def __init__(self, model_type: str, n_s_ls: Sequence[int], n_a_ls: Sequence[int], n_w_ls: Sequence[int],
                 obs_off: Sequence[int], n_obs: int, n_fc: int = 0, n_ft: int = 0, n_h: int = 0, max_na: int | None = None):
        if model_type not in ("lr", "dqn"):
            raise ValueError("model_type must be 'lr' or 'dqn' (got %r)" % (model_type,))
        self.model_type = model_type
        self.A = len(n_s_ls)
        self.n_s = np.asarray(n_s_ls, np.int32)
        self.n_a = np.asarray(n_a_ls, np.int32)
        self.n_w = np.asarray(n_w_ls, np.int32) if model_type == "dqn" else np.zeros(self.A, np.int32)
        self.obs_off = np.asarray(obs_off, np.int32)[:self.A].copy()
        self.n_obs = int(n_obs)
        self.max_na = int(max_na or self.n_a.max())
        dqn = model_type == "dqn"
        self.n_fc, self.n_h = (int(n_fc), int(n_h)) if dqn else (0, 0)
        self.n_ft = int(n_ft) if dqn and (self.n_w > 0).any() else 0
        self.shapes = []                      # per agent: {name: shape} in flat order
        for n in self.OFF.values():
            setattr(self, n, np.zeros(self.A, np.int64))
        off = 0
        for i in range(self.A):
            n_s, n_a, n_w = int(self.n_s[i]), int(self.n_a[i]), int(self.n_w[i])
            if dqn:
                shp = {"q_fcw/w": (n_s - n_w, self.n_fc), "q_fcw/b": (self.n_fc,)}
                if n_w > 0:
                    shp.update({"q_fct/w": (n_w, self.n_ft), "q_fct/b": (self.n_ft,)})
                width = self.n_fc + (self.n_ft if n_w > 0 else 0)
                shp.update({"q_fc_0/w": (width, self.n_h), "q_fc_0/b": (self.n_h,), "q/w": (self.n_h, n_a), "q/b": (n_a,)})
            else:
                shp = {"q/w": (n_s, n_a), "q/b": (n_a,)}
            self.shapes.append(shp)
            for k, s in shp.items():
                getattr(self, self.OFF[k])[i] = off
                off += int(np.prod(s))
            for k, n in self.OFF.items():     # layers the agent lacks: zero length at the end of its block
                if k not in shp:
                    getattr(self, n)[i] = off
        self.n_params = off

    @classmethod
    def from_iql(cls, model, obs_off, n_obs, max_na=None) -> "QLayout":
        """The layout of an `agents/models.py:IQL`, with the widths read from its tensors (not from the config)."""
        nets = model.nets
        if model.model_type == "dqn":
            n_fc = int(nets[0]["q_fcw/w"].shape[1])
            n_h = int(nets[0]["q_fc_0/w"].shape[1])
            with_t = [p for p in nets if "q_fct/w" in p]
            n_ft = int(with_t[0]["q_fct/w"].shape[1]) if with_t else 0
        else:
            n_fc = n_ft = n_h = 0
        lay = cls(model.model_type, model.n_s_ls, model.n_a_ls, model.n_w_ls, obs_off, n_obs, n_fc=n_fc, n_ft=n_ft,
                  n_h=n_h, max_na=max_na)
        for i, p in enumerate(nets):
            got = {k: tuple(v.shape) for k, v in p.items()}
            if got != {k: tuple(s) for k, s in lay.shapes[i].items()}:
                raise ValueError("IQL agent %d: tensor shapes %s differ from the layout's %s" % (i, got, lay.shapes[i]))
        return lay

    def pack(self, nets):
        """`IQL.nets` (a list of {name: tensor}) -> the flat float32 vector: a torch tensor on the tensors' device when
        they are torch tensors (no host round trip), else a numpy array."""
        parts = [nets[i][k] for i in range(self.A) for k in self.shapes[i]]
        if parts and hasattr(parts[0], "detach"):
            import torch
            return torch.cat([t.detach().reshape(-1).to(torch.float32) for t in parts])
        return np.concatenate([np.asarray(t, np.float32).reshape(-1) for t in parts]).astype(np.float32)

    def views(self, flat):
        """Per agent {name: view} into a flat vector (numpy or torch), the inverse of pack()."""
        out = []
        for i in range(self.A):
            v = {}
            for k, s in self.shapes[i].items():
                o = int(getattr(self, self.OFF[k])[i])
                v[k] = flat[o:o + int(np.prod(s))].reshape(s)
            out.append(v)
        return out

    def as_c(self) -> CQDims:
        c = CQDims()
        c.n_agents, c.n_obs, c.max_na = self.A, self.n_obs, self.max_na
        c.model = 1 if self.model_type == "dqn" else 0
        c.n_fc, c.n_ft, c.n_h = self.n_fc, self.n_ft, self.n_h
        for name in ("obs_off", "n_s", "n_w", "n_a"):
            setattr(c, name, getattr(self, name).ctypes.data_as(C.POINTER(C.c_int32)))
        for name in self.OFF.values():
            setattr(c, name, getattr(self, name).ctypes.data_as(C.POINTER(C.c_int64)))
        c.n_params = self.n_params
        c._keep = self
        return c
