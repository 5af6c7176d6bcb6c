"""CPU ORACLE of the learner math (test infrastructure only): float64 torch/numpy restatement of

  fc / lstm              reference agents/utils.py:66-74, 88-116  (gate order i,f,o,u; done masks c,h)
  FPLstmACPolicy         reference agents/policies.py:191-211     (h = concat(fcw, fcf, fct))
  FcACPolicy             reference agents/policies.py:214-256     (h = relu(fc(concat(fcw, fct))), no state)
  A2C loss               reference agents/policies.py:41-52
  n-step returns         reference agents/utils.py:202-214
  clip + RMSProp         reference agents/policies.py:54-61 (TF1: rms slot starts at 1, eps inside sqrt)

Pinned against the reference where it is pure Python (OnPolicyBuffer, Scheduler: tests/golden/buffers.npz);
the TF1 graph math itself cannot run here (TensorFlow 1.12 is absent) -> parity of those ops is against this
restatement with autograd as the differentiation oracle.
"""
import numpy as np
import torch


def nstep_returns(rs, vs, dones_post, R, gamma):
    """agents/utils.py:202-214."""
    Rs, Advs = [], []
    for r, v, done in zip(rs[::-1], vs[::-1], dones_post[::-1]):
        R = r + gamma * R * (1. - done)
        Rs.append(R)
        Advs.append(R - v)
    return np.array(Rs[::-1]), np.array(Advs[::-1])


def _obs_blocks(lay, u, obs):
    """(wave, wait, fingerprint) input slices of unit u."""
    a = u // 2
    o0 = int(lay.obs_off[a]); nw, nt, nf = int(lay.n_wave[a]), int(lay.n_wait[a]), int(lay.n_fp[a])
    return obs[..., o0:o0 + nw], obs[..., o0 + nw:o0 + nw + nt], obs[..., o0 + nw + nt:o0 + nw + nt + nf]


def fc_front(v, lay, u, obs):
    """x = concat(fcw, fcf, fct) of unit u (agents/policies.py:191-211)."""
    wave, wait, fp = _obs_blocks(lay, u, obs)
    parts = [torch.relu(wave @ v["fcw_w%d" % u] + v["fcw_b%d" % u])]
    if lay.ff > 0:
        parts.append(torch.relu(fp @ v["fcf_w%d" % u] + v["fcf_b%d" % u]))
    if lay.ft > 0:
        parts.append(torch.relu(wait @ v["fct_w%d" % u] + v["fct_b%d" % u]))
    return torch.cat(parts, -1)


def unit_forward(v, lay, u, obs, dones, c, h):
    """obs [T, R, n_obs] -> (pi or value [T, R, ...], H [T, R, h], final c, h).  float64 torch."""
    a = u // 2
    x = fc_front(v, lay, u, obs)
    H = lay.h
    if not getattr(lay, "recurrent", True):      # FcACPolicy: one more fc layer instead of the LSTM
        Hs = torch.relu(x @ v["wx"][u] + v["bl"][u])
        n_out = int(lay.n_a[a]) if u % 2 == 0 else 1
        out = Hs @ v["wo"][u][:, :n_out] + v["bo"][u][:n_out]
        out = torch.softmax(out, -1) if u % 2 == 0 else out.squeeze(-1)
        return out, Hs, c, h
    hs = []
    for t in range(obs.shape[0]):
        keep = 1.0 - dones[t]
        c = c * keep; h = h * keep
        z = x[t] @ v["wx"][u] + h @ v["wh"][u] + v["bl"][u]
        i, f, o, g = (torch.sigmoid(z[:, :H]), torch.sigmoid(z[:, H:2 * H]), torch.sigmoid(z[:, 2 * H:3 * H]),
                      torch.tanh(z[:, 3 * H:]))
        c = f * c + i * g
        h = o * torch.tanh(c)
        hs.append(h)
    Hs = torch.stack(hs)
    n_out = int(lay.n_a[a]) if u % 2 == 0 else 1
    out = Hs @ v["wo"][u][:, :n_out] + v["bo"][u][:n_out]
    if u % 2 == 0:
        out = torch.softmax(out, -1)
    else:
        out = out.squeeze(-1)
    return out, Hs, c, h


def a2c_loss(P, lay, obs, acts, Rs, Advs, dones, c0, h0, v_coef, beta):
    """Sum over agents of the per-agent loss averaged over (t, replica).  Returns (loss, per-agent parts)."""
    v = lay.views(P)
    total = 0.0
    parts = []
    for a in range(lay.A):
        pi, _, _, _ = unit_forward(v, lay, 2 * a, obs, dones, c0[2 * a], h0[2 * a])
        val, _, _, _ = unit_forward(v, lay, 2 * a + 1, obs, dones, c0[2 * a + 1], h0[2 * a + 1])
        log_pi = torch.log(torch.clamp(pi, 1e-10, 1.0))
        ent = -(pi * log_pi).sum(-1)
        lp_a = torch.gather(log_pi, -1, acts[..., a].long().unsqueeze(-1)).squeeze(-1)
        pl = -(lp_a * Advs[..., a]).mean()
        vl = ((Rs[..., a] - val) ** 2).mean() * 0.5 * v_coef
        el = -ent.mean() * beta
        total = total + pl + vl + el
        parts.append((pl.item(), vl.item(), el.item()))
    return total, parts


def clip_rmsprop(P, G, MS, agent_of, max_norm, lr, alpha, eps, n_agents):
    P, G, MS = P.copy(), G.copy(), MS.copy()
    norms = np.zeros(n_agents)
    for a in range(n_agents):
        m = agent_of == a
        nrm = np.sqrt((G[m].astype(np.float64) ** 2).sum())
        norms[a] = nrm
        g = G[m] * (max_norm / max(nrm, max_norm) if max_norm > 0 else 1.0)
        MS[m] = alpha * MS[m] + (1 - alpha) * g * g
        P[m] = P[m] - lr * g / np.sqrt(MS[m] + eps)
    return P, MS, norms


# ------------------------------------------------------------------------------------------------
# The update from the bf16 activation store (BatchedA2C.backward with use_tc and store_acts), in float64.
# Per chunk of rc replicas starting at r0 the kernels read the store [U][T][rc][w] (X, gate activations i, f, o, u, c, h),
# obs / actions / returns / advantages, the fp32 parameters, c_bw / h_bw rows r0 .. r0 + rc and done_pre, and run
#   heads_loss -> BPTT (dZ) -> [X | Hp | 1]^T dZ and dX = dZ . Wx^T -> fc front-end gradients.
# These functions take exactly those inputs and return float64 results.  With round_bf16 they round to bf16 where the
# kernels do and nowhere else: the Wh / Wx operand images, dz before the recurrent product and as the dZ operand, dX as
# stored, obs and h0 as GEMM operands.  round_bf16=False gives the exact gradient of a2c_loss through the same store.

def bf16(x):
    """Round to the nearest bf16 (ties to even) and back to x's dtype."""
    return x.to(torch.bfloat16).to(x.dtype)


def tf32(x):
    """Round to the nearest TF32 value (11 significant bits, ties to even) in x's dtype: the operand rounding of a TF32
    tensor-core product.  A model of it only: how the library rounds its TF32 operands is not specified."""
    m, e = torch.frexp(x)
    return torch.ldexp(torch.round(m * 2048.0) / 2048.0, e)


def store_forward(v, lay, u, obs, dones, c0, h0):
    """Float64 forward of unit u in the activation-store layout: obs [T, rc, n_obs], c0 / h0 [rc, h] ->
    (X [T, rc, dx], gate activations [T, rc, 4h] in the order i, f, o, u, c [T, rc, h], h [T, rc, h])."""
    x = fc_front(v, lay, u, obs)
    H = lay.h
    gs, cs, hs = [], [], []
    c, h = c0, h0
    for t in range(obs.shape[0]):
        keep = 1.0 - float(dones[t])
        c = c * keep; h = h * keep
        z = x[t] @ v["wx"][u] + h @ v["wh"][u] + v["bl"][u]
        g = torch.cat([torch.sigmoid(z[:, :3 * H]), torch.tanh(z[:, 3 * H:])], -1)
        c = g[:, H:2 * H] * c + g[:, :H] * g[:, 3 * H:]
        h = g[:, 2 * H:3 * H] * torch.tanh(c)
        gs.append(g); cs.append(c); hs.append(h)
    return x, torch.stack(gs), torch.stack(cs), torch.stack(hs)


def heads_ref(lay, v, a, H_pi, H_v, act, Rs, Adv, scale, v_coef, beta):
    """Loss gradients at the heads of agent a (tscl_heads_loss) over rows [M]: H_pi / H_v [M, h], act / Rs / Adv [M].
    Returns dH_pi / dH_v [M, h], the head gradients wo_pi [h, n_a], bo_pi [n_a], wo_v [h], bo_v [] and the loss sums
    (policy, value, entropy) times `scale` (BatchedA2C.stats for agent 0).  TF clip semantics:
    d log(clip(p, 1e-10, 1)) / dp = 0 outside [1e-10, 1] (agents/policies.py:47)."""
    na = int(lay.n_a[a])
    Wp, bp = v["wo"][2 * a][:, :na], v["bo"][2 * a][:na]
    wv, bv = v["wo"][2 * a + 1][:, 0], v["bo"][2 * a + 1][0]
    val = H_v @ wv + bv
    dv = scale * v_coef * (val - Rs)
    pi = torch.softmax(H_pi @ Wp + bp, -1)
    m = ((pi >= 1e-10) & (pi <= 1.0)).to(pi.dtype)
    lp = torch.log(pi.clamp(1e-10, 1.0))
    ent = -(pi * lp).sum(-1)
    onehot = torch.nn.functional.one_hot(act.long(), na).to(pi.dtype)
    m_at = (m * onehot).sum(-1)
    dl = scale * (-(Adv * m_at)[:, None] * (onehot - pi)
                  + beta * pi * (lp + m + ent[:, None] - (pi * m).sum(-1, keepdim=True)))
    lp_at = (lp * onehot).sum(-1)
    stats = scale * torch.stack([-(lp_at * Adv).sum(), 0.5 * v_coef * ((Rs - val) ** 2).sum(), -beta * ent.sum()])
    return dict(dH_pi=dl @ Wp.T, dH_v=dv[:, None] * wv[None, :], wo_pi=H_pi.T @ dl, bo_pi=dl.sum(0), wo_v=H_v.T @ dv,
                bo_v=dv.sum(), stats=stats)


def bptt_ref(gates, c, c0, dH, dones, wh, round_bf16=True, c_prev=None):
    """BPTT through the LSTM from stored activations, t = T-1 .. 0 (tscl_lstm_seq_bwd_tc).  gates [..., T, rc, 4h]
    (i, f, o, u activated), c [..., T, rc, h], c0 [..., rc, h] (c_bw rows r0 .. r0 + rc), dH [..., T, rc, h],
    wh [..., h, 4h]; the leading dimensions are units.  c_{t-1} and the carries into step t-1 are masked by
    1 - done[t].  Returns dZ [..., T, rc, 4h] unrounded; the recurrent product is bf16(dz) . bf16(Wh)^T with round_bf16.
    `c_prev` [..., T, rc, h] replaces (c0, c_0 .. c_{T-2}) as the previous cell state (tests use it to plant defects)."""
    H, T = c.shape[-1], c.shape[-3]
    whT = (bf16(wh) if round_bf16 else wh).transpose(-1, -2)
    dZ = torch.empty_like(gates)
    dc = torch.zeros_like(c0)
    dhc = torch.zeros_like(c0)
    for t in range(T - 1, -1, -1):
        keep = 1.0 - float(dones[t])
        g = gates[..., t, :, :]
        i, f, o, u = g[..., :H], g[..., H:2 * H], g[..., 2 * H:3 * H], g[..., 3 * H:]
        if c_prev is not None:
            cp = c_prev[..., t, :, :] * keep
        else:
            cp = (c[..., t - 1, :, :] if t > 0 else c0) * keep
        dh = dH[..., t, :, :] + dhc
        tc = torch.tanh(c[..., t, :, :])
        dcc = dc + dh * o * (1.0 - tc * tc)
        dz = torch.cat([dcc * u * i * (1.0 - i), dcc * cp * f * (1.0 - f), dh * tc * o * (1.0 - o),
                        dcc * i * (1.0 - u * u)], -1)
        dZ[..., t, :, :] = dz
        dc = dcc * f * keep
        dhc = ((bf16(dz) if round_bf16 else dz) @ whT) * keep
    return dZ


def lstm_grads_ref(X, Hs, h0, dones, dZ, wx, round_bf16=True, round_operands=False, dx_product="bf16", dx_bf16=True):
    """LSTM weight gradients [X | Hp | 1]^T dZ and dX = dZ . Wx^T (tscl_wgrad_tc, tscl_dx_tc).  X [..., T, rc, dx],
    Hs [..., T, rc, h] (store), h0 [..., rc, h] (h_bw rows r0 .. r0 + rc), dZ [..., T, rc, 4h], wx [..., dx, 4h].
    Hp[t] = (1 - done[t]) * (h[t-1], or h0 at t = 0).  Returns (wx, wh, bl, dX [..., T, rc, dx]).
    With round_bf16 (nothing is rounded without it):
      round_operands  X and all of Hp are rounded to bf16 as GEMM operands (the recompute path: wgrad_tc_kernel converts
                      its fp32 X / Hp; on the store path they are bf16 already and only h0 is rounded);
      dx_product      operands of dX: "bf16" bf16(dZ) . bf16(Wx)^T (the store path's tensor-core kernels), "fp32" the
                      unrounded fp32 dZ . Wx^T, "tf32" both rounded to TF32 (torch.bmm with TF32 allowed);
    dX is then rounded to bf16, where the fc weight-gradient kernel converts it (not with dx_bf16=False: the SIMT
    tscl_fc_bwd reads it in fp32)."""
    keep = (1.0 - torch.as_tensor([float(d) for d in dones], dtype=X.dtype, device=X.device))[:, None, None]
    h0r = bf16(h0) if round_bf16 else h0
    Hp = torch.cat([h0r.unsqueeze(-3), Hs[..., :-1, :, :]], -3) * keep
    if round_bf16 and round_operands:
        X, Hp = bf16(X), bf16(Hp)
    Z = bf16(dZ) if round_bf16 else dZ
    flat = lambda t_: t_.reshape(*t_.shape[:-3], -1, t_.shape[-1])
    Zf = flat(Z)
    gwx = flat(X).transpose(-1, -2) @ Zf
    gwh = flat(Hp).transpose(-1, -2) @ Zf
    rnd = {"bf16": bf16, "fp32": lambda t_: t_, "tf32": tf32}[dx_product if round_bf16 else "fp32"]
    dX = (Z if dx_product == "bf16" else rnd(dZ)) @ rnd(wx).transpose(-1, -2).unsqueeze(-3)
    return gwx, gwh, Zf.sum(-2), (bf16(dX) if round_bf16 and dx_bf16 else dX)


def fc_grads_ref(lay, u, obs, X, dX, round_bf16=True):
    """fc front-end gradients of unit u (tscl_fc_bwd_tc): obs [T, rc, n_obs] (the chunk's rows), X / dX [T, rc, dx].
    relu mask from X.  Returns {view name: gradient} for the fcw / fcf / fct weights and biases of u."""
    wave, wait, fp = _obs_blocks(lay, u, bf16(obs) if round_bf16 else obs)
    dd = (dX * (X > 0)).reshape(-1, lay.dx)
    out = {}
    for name, inp, c0, w in (("fcw", wave, 0, lay.fw), ("fcf", fp, lay.fw, lay.ff), ("fct", wait, lay.fw + lay.ff, lay.ft)):
        if w == 0:
            continue
        d_ = dd[:, c0:c0 + w]
        out["%s_w%d" % (name, u)] = inp.flatten(0, -2).T @ d_           # flatten: the block may be empty
        out["%s_b%d" % (name, u)] = d_.sum(0)
    return out


def update_ref(lay, P, store, obs, act, Rs, Adv, c_bw, h_bw, dones, scale, v_coef, beta, chunk, round_bf16=True,
               agents_per_group=None, store_units=False, round_operands=False, dx_product="bf16", agents=None,
               fc_fp32=False):
    """Flat gradient G (float64) of one update from the activation store, summed over the chunks r0 = 0, chunk, ...
    P: fp32 parameters (any float tensor); store(ci) -> (st_x, st_g, st_c, st_h) of chunk ci, each [U][T][rc][w], or
    with `store_units` store(ci, us) -> the same for the unit slice `us` only (lets a caller compute the store of one agent
    group at a time, e.g. store_group below for the recompute path);
    obs [T, R, n_obs], act / Rs / Adv [T, R, A], c_bw / h_bw [U, R, h], dones = done_pre [T].  Work runs on P's device,
    `agents_per_group` agents at a time (bounds the float64 working set); `agents` (a range) restricts the sum to those
    agents.  round_operands / dx_product: see lstm_grads_ref (the defaults are the store path's rounding; the recompute
    path is round_operands=True with dx_product "fp32" or "tf32").  `fc_fp32`: the fc front-end gradients from fp32 obs and
    dX (the store path of a layout without a spare bias slot: dX by torch.bmm, then the SIMT tscl_fc_bwd).
    Returns (G, agent-0 stats)."""
    f64 = dict(dtype=torch.float64, device=P.device)
    v = lay.views(P.to(torch.float64))
    G = torch.zeros(lay.n_params, **f64)
    gv = lay.views(G)
    stats = torch.zeros(3, **f64)
    T, R, A, hd = obs.shape[0], obs.shape[1], lay.A, lay.h
    grp = agents_per_group or A
    agents = agents if agents is not None else range(A)
    for ci, r0 in enumerate(range(0, R, chunk)):
        rc = min(chunk, R - r0)
        st = None if store_units else store(ci)
        ob = obs[:, r0:r0 + rc].to(**f64)
        for a0 in range(agents.start, agents.stop, grp):
            a1 = min(agents.stop, a0 + grp)
            us = slice(2 * a0, 2 * a1)
            X, Gt, Cs, Hs = (s.to(**f64) for s in store(ci, us)) if store_units else (s[us].to(**f64) for s in st)
            dH = torch.empty_like(Hs)
            for a in range(a0, a1):
                k = 2 * (a - a0)
                hr = heads_ref(lay, v, a, Hs[k].reshape(-1, hd), Hs[k + 1].reshape(-1, hd),
                               act[:, r0:r0 + rc, a].reshape(-1).to(P.device), Rs[:, r0:r0 + rc, a].reshape(-1).to(**f64),
                               Adv[:, r0:r0 + rc, a].reshape(-1).to(**f64), scale, v_coef, beta)
                dH[k] = hr["dH_pi"].reshape(T, rc, hd)
                dH[k + 1] = hr["dH_v"].reshape(T, rc, hd)
                na = int(lay.n_a[a])
                gv["wo"][2 * a][:, :na] += hr["wo_pi"]
                gv["bo"][2 * a][:na] += hr["bo_pi"]
                gv["wo"][2 * a + 1][:, 0] += hr["wo_v"]
                gv["bo"][2 * a + 1][0] += hr["bo_v"]
                if a == 0:
                    stats += hr["stats"]
            c0 = c_bw[us, r0:r0 + rc].to(**f64)
            h0 = h_bw[us, r0:r0 + rc].to(**f64)
            dZ = bptt_ref(Gt, Cs, c0, dH, dones, v["wh"][us], round_bf16)
            del dH, Gt, Cs
            gwx, gwh, gbl, dX = lstm_grads_ref(X, Hs, h0, dones, dZ, v["wx"][us], round_bf16, round_operands, dx_product,
                                               dx_bf16=not fc_fp32)
            del dZ
            gv["wx"][us] += gwx
            gv["wh"][us] += gwh
            gv["bl"][us] += gbl
            for k, u in enumerate(range(us.start, us.stop)):
                for name, g in fc_grads_ref(lay, u, ob, X[k], dX[k], round_bf16 and not fc_fp32).items():
                    gv[name] += g
            del X, Hs, dX
    return G, stats


def bptt_mutations(gates, c, c_state, r0, dH, dones):
    """Arguments of bptt_ref (without wh) for the correct chunk and for six planted defects of a BPTT kernel:
    returns ({gates, c, c0, dH, dones}, {defect name: the same with the defect}).  c_state [..., R, h] is c_bw; the chunk
    starts at replica r0 > 0."""
    rc, H, T = c.shape[-2], c.shape[-1], len(dones)
    ok = dict(gates=gates, c=c, c0=c_state[..., r0:r0 + rc, :], dH=dH, dones=[float(d) for d in dones])
    swapped = torch.cat([gates[..., H:2 * H], gates[..., :H], gates[..., 2 * H:]], -1)
    late = lambda x: torch.cat([torch.zeros_like(x[..., :1, :, :]), x[..., :-1, :, :]], -3)
    return ok, {
        "c0 from row r instead of r0 + r": dict(ok, c0=c_state[..., :rc, :]),
        "done one step late": dict(ok, dones=[0.0] + ok["dones"][:-1]),
        "done ignored": dict(ok, dones=[0.0] * T),
        "i and f gates swapped": dict(ok, gates=swapped),
        "c_t in place of c_{t-1}": dict(ok, c_prev=c),
        "dH one step late": dict(ok, dH=late(dH)),
    }


# ------------------------------------------------------------------------------------------------
# The recompute update (BatchedA2C.backward without the activation store): per chunk the forward is recomputed in fp32
# (tscl_fc_embed, X . Wx + bl, tscl_lstm_seq_fwd from c_bw / h_bw rows r0 .. r0 + rc), then heads_loss -> BPTT with fp32
# gates / c (dZ written fp32; the recurrent product is bf16(dz) . bf16(Wh)^T as on the store path) -> wgrad_tc_kernel,
# which rounds its fp32 X / Hp / dZ operands to bf16 -> dX = dZ . Wx^T in fp32 or TF32 -> fc weight gradients from
# bf16(obs) and bf16(dX * (X > 0)).  Its float64 reference is update_ref over the float64 forward (store_group) with
# round_operands=True and dx_product "fp32" / "tf32".

def store_group(v, lay, us, obs, dones, c0, h0):
    """store_forward of the units of slice `us`, stacked: obs [T, rc, n_obs], c0 / h0 [U, rc, h] (all units, the chunk's
    rows) -> (X, gates, c, h), each [len(us)][T][rc][w]."""
    st = [store_forward(v, lay, u, obs, dones, c0[u], h0[u]) for u in range(us.start, us.stop)]
    return tuple(torch.stack([s[k] for s in st]) for k in range(4))


def recompute_mutations(obs, c_state, h_state, dones, r0, rc):
    """Forward inputs of store_group for the chunk of rc replicas at r0, correct and with four planted defects of the
    recompute forward: returns ({obs, dones, c0, h0}, {defect name: the same with the defect}).  obs [T + 1, R, n_obs]
    are the rollout's observation slots (slot T is the next observation), c_state / h_state [U, R, h] are c_bw / h_bw."""
    T = len(dones)
    ok = dict(obs=obs[:T, r0:r0 + rc], dones=[float(d) for d in dones], c0=c_state[:, r0:r0 + rc],
              h0=h_state[:, r0:r0 + rc])
    return ok, {
        "recompute from zero state": dict(ok, c0=torch.zeros_like(ok["c0"]), h0=torch.zeros_like(ok["h0"])),
        "state from row r instead of r0 + r": dict(ok, c0=c_state[:, :rc], h0=h_state[:, :rc]),
        "done one step late": dict(ok, dones=[0.0] + ok["dones"][:-1]),
        "obs slot t + 1 instead of t": dict(ok, obs=obs[1:T + 1, r0:r0 + rc]),
    }


# ------------------------------------------------------------------------------------------------
# The FcACPolicy update (BatchedFcA2C.backward): per chunk fc front end -> H = relu(X . wx + bl) (tscl_fc_hidden_fwd) ->
# heads_loss -> dHm = dH * (H > 0), dX = dHm . wx^T, bl / wx gradients (tscl_fc_hidden_bwd, all fp32) -> fc weight
# gradients from bf16(obs) and bf16(dX * (X > 0)) (tscl_fc_bwd_tc).

FC_DEFECTS = ("hidden relu mask ignored", "bias gradient from unmasked dH",
              "value unit uses the policy unit's hidden weights")


def fc_update_ref(lay, P, obs, act, Rs, Adv, scale, v_coef, beta, chunk, round_bf16=False, agents=None, defect=None):
    """Flat gradient G (float64) of one FcACPolicy update, summed over the chunks r0 = 0, chunk, ...: P fp32 parameters
    of a PolicyLayout(recurrent=False), obs [T, R, n_obs], act / Rs / Adv [T, R, A].  round_bf16: obs and dX rounded to
    bf16 where the tensor-core fc weight-gradient kernel reads them (nothing else is rounded: the other kernels are fp32).
    `agents` (a range) restricts the sum to those agents; `defect` plants one of FC_DEFECTS.  Returns (G, agent-0 stats)."""
    assert defect is None or defect in FC_DEFECTS, defect
    f64 = dict(dtype=torch.float64, device=P.device)
    v = lay.views(P.to(torch.float64))
    G = torch.zeros(lay.n_params, **f64)
    gv = lay.views(G)
    stats = torch.zeros(3, **f64)
    T, R, hd = obs.shape[0], obs.shape[1], lay.h
    for r0 in range(0, R, chunk):
        rc = min(chunk, R - r0)
        ob = obs[:, r0:r0 + rc].to(**f64)
        for a in (agents if agents is not None else range(lay.A)):
            units = (2 * a, 2 * a + 1)
            # hidden weights each unit's kernels read (the third defect: the value unit reads the policy unit's)
            w_of = {u: v["wx"][2 * a if defect == FC_DEFECTS[2] else u] for u in units}
            X = {u: fc_front(v, lay, u, ob).reshape(-1, lay.dx) for u in units}
            H = {u: torch.relu(X[u] @ w_of[u] + v["bl"][u]) for u in units}
            sl = lambda t_: t_[:, r0:r0 + rc, a].reshape(-1)
            hr = heads_ref(lay, v, a, H[units[0]], H[units[1]], sl(act).to(P.device), sl(Rs).to(**f64),
                           sl(Adv).to(**f64), scale, v_coef, beta)
            na = int(lay.n_a[a])
            gv["wo"][units[0]][:, :na] += hr["wo_pi"]
            gv["bo"][units[0]][:na] += hr["bo_pi"]
            gv["wo"][units[1]][:, 0] += hr["wo_v"]
            gv["bo"][units[1]][0] += hr["bo_v"]
            if a == 0:
                stats += hr["stats"]
            for u, dH in zip(units, (hr["dH_pi"], hr["dH_v"])):
                dHm = dH if defect == FC_DEFECTS[0] else dH * (H[u] > 0)
                gv["wx"][u] += X[u].T @ dHm
                gv["bl"][u] += (dH if defect == FC_DEFECTS[1] else dHm).sum(0)
                dX = (dHm @ w_of[u].T).reshape(T, rc, lay.dx)
                for name, g in fc_grads_ref(lay, u, ob, X[u].reshape(T, rc, lay.dx), bf16(dX) if round_bf16 else dX,
                                            round_bf16).items():
                    gv[name] += g
    return G, stats
