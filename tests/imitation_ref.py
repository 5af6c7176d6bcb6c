"""Float64 reference of the imitation term of the A2C update (BatchedA2C(teacher=...), DESIGN §5 Imitation).

For a row with logits z, pi = softmax(z), teacher action b and coefficient lam, the loss gains
-lam * log clip(pi_b, 1e-10, 1) * scale; its gradient at the logits is scale * lam * (pi_j - [j == b]) when pi_b is not
clipped and 0 when it is.  That is the A2C policy-gradient term with Adv := lam and act := b, and the backward of the
update is linear in the logits' gradient, so the references below are the oracle's (oracle/learner_ref.py) A2C
references plus the same references run once more with (act := teach, Adv := lam, v_coef = beta = 0).
"""
import torch

from oracle.learner_ref import fc_update_ref, heads_ref, update_ref


def imit_loss(logits, teach, lam, scale):
    """(loss, cross-entropy) of rows `logits` [M, na] toward `teach` [M]: -lam * scale * sum log clip(pi_b, 1e-10, 1) and
    scale * sum -log clip(pi_b, 1e-10, 1), differentiable with torch.clamp's zero gradient outside [1e-10, 1]."""
    pi = torch.softmax(logits, -1)
    lp_b = torch.log(pi.gather(1, teach.long()[:, None])[:, 0].clamp(1e-10, 1.0))
    return -lam * scale * lp_b.sum(), -scale * lp_b.sum()


def imit_dlog(logits, teach, lam, scale):
    """The closed form of d imit_loss / d logits: scale * lam * (pi - onehot(b)) on rows where pi_b lies in [1e-10, 1]."""
    pi = torch.softmax(logits, -1)
    onehot = torch.nn.functional.one_hot(teach.long(), logits.shape[1]).to(pi.dtype)
    pb = (pi * onehot).sum(-1)
    keep = ((pb >= 1e-10) & (pb <= 1.0)).to(pi.dtype)
    return scale * lam * keep[:, None] * (pi - onehot)


def heads_imit_ref(lay, v, a, H_pi, H_v, act, teach, Rs, Adv, scale, v_coef, beta, lam):
    """heads_ref with the imitation term (tscl_heads_loss_imit): the same keys, `stats` with a 4th entry, agent a's
    unweighted cross-entropy sum times scale."""
    r = heads_ref(lay, v, a, H_pi, H_v, act, Rs, Adv, scale, v_coef, beta)
    t = heads_ref(lay, v, a, H_pi, H_v, teach, Rs, torch.full_like(Adv, lam), scale, 0.0, 0.0)
    out = dict(r)
    for key in ("dH_pi", "wo_pi", "bo_pi"):
        out[key] = r[key] + t[key]
    na = int(lay.n_a[a])
    logits = H_pi @ v["wo"][2 * a][:, :na] + v["bo"][2 * a][:na]
    ce = imit_loss(logits, teach, lam, scale)[1]
    out["stats"] = torch.cat([r["stats"], ce.reshape(1)])
    return out


def update_imit_ref(lay, P, store, obs, act, teach, Rs, Adv, c_bw, h_bw, dones, scale, v_coef, beta, lam, chunk, **kw):
    """update_ref of an update with a teacher: (G float64, agent-0 stats [4])."""
    G, st = update_ref(lay, P, store, obs, act, Rs, Adv, c_bw, h_bw, dones, scale, v_coef, beta, chunk, **kw)
    Gt, st_t = update_ref(lay, P, store, obs, teach, Rs, torch.full_like(Adv, lam), c_bw, h_bw, dones, scale, 0.0, 0.0,
                          chunk, **kw)
    ce = st_t[0] / lam if lam else torch.zeros_like(st_t[0])
    return G + Gt, torch.cat([st, ce.reshape(1)])


def fc_update_imit_ref(lay, P, obs, act, teach, Rs, Adv, scale, v_coef, beta, lam, chunk, **kw):
    """fc_update_ref of an FC-policy update with a teacher: (G float64, agent-0 stats [4])."""
    G, st = fc_update_ref(lay, P, obs, act, Rs, Adv, scale, v_coef, beta, chunk, **kw)
    Gt, st_t = fc_update_ref(lay, P, obs, teach, Rs, torch.full_like(Adv, lam), scale, 0.0, 0.0, chunk, **kw)
    ce = st_t[0] / lam if lam else torch.zeros_like(st_t[0])
    return G + Gt, torch.cat([st, ce.reshape(1)])
