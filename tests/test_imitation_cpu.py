"""CPU: imitation of a signal controller in the A2C update (BatchedA2C(teacher=...), DESIGN §5 Imitation).

- The float64 reference (tests/imitation_ref.py) against autograd in float64: the closed-form gradient of the
  imitation term, with rows where pi_b is clipped (zero gradient) and rows where b equals the sampled action; and the
  heads' gradients of the whole loss (A2C + imitation) through the composed reference.
- Every refusal of the [MODEL_CONFIG] imitation keys, each naming its key, before any directory is made.
- The defaults and the values of the lam schedule, with imitation_ratio.
- Sweep rules: the imitation keys may differ between members, the teacher may not.
- The summary tags of a 5-column record.
"""
import configparser

import numpy as np
import pytest
import torch

from tests.imitation_ref import heads_imit_ref, imit_dlog, imit_loss
from tests.test_train_driver_gpu import _ini


def _rows(M, na, seed, clip_col=1):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(M, na, generator=g, dtype=torch.float64) * 2
    logits[::3, clip_col] = -40.0                               # pi < 1e-10: clipped
    act = torch.randint(0, na, (M,), generator=g)
    teach = torch.randint(0, na, (M,), generator=g)
    teach[::3] = clip_col                                       # the teacher's action is clipped on these rows
    teach[1::4] = act[1::4]                                     # b == a
    return logits, act, teach


@pytest.mark.parametrize("na", [2, 5, 8])
def test_imitation_gradient_against_autograd(na):
    logits, _, teach = _rows(96, na, seed=na)
    lam, scale = 0.7, 1.0 / 96
    z = logits.clone().requires_grad_(True)
    loss, ce = imit_loss(z, teach, lam, scale)
    (grad,) = torch.autograd.grad(loss, z)
    ref = imit_dlog(logits, teach, lam, scale)
    torch.testing.assert_close(grad, ref, rtol=1e-12, atol=1e-15)
    clipped = torch.softmax(logits, -1).gather(1, teach[:, None])[:, 0] < 1e-10
    assert clipped.sum() >= 20 and bool((ref[clipped] == 0).all())
    assert bool((ref[~clipped].abs().sum(1) > 0).all())
    # the unweighted cross-entropy: lam does not scale it
    assert float(loss.detach()) == pytest.approx(lam * float(ce.detach()), rel=1e-12)
    torch.testing.assert_close(ce, -scale * torch.log(torch.softmax(logits, -1).gather(1, teach[:, None])[:, 0]
                                                      .clamp(1e-10, 1.0)).sum())


class _Lay:
    def __init__(self, n_a):
        self.n_a = np.asarray(n_a)


@pytest.mark.parametrize("beta,lam", [(0.01, 0.5), (0.0, 2.0), (0.05, 0.0)])
def test_heads_reference_against_autograd_of_the_whole_loss(beta, lam):
    """heads_imit_ref's dH (both heads) and loss sums = autograd of the A2C loss of agents/policies.py:41-52 plus the
    imitation term, in float64, with the advantage held constant."""
    M, h, na, v_coef = 120, 16, 5, 0.5
    g = torch.Generator().manual_seed(5)
    f64 = dict(dtype=torch.float64)
    Wp, bp = torch.randn(h, na, generator=g, **f64), torch.randn(na, generator=g, **f64)
    bp[1] = -40.0                                               # pi_1 < 1e-10 everywhere
    wv, bv = torch.randn(h, 1, generator=g, **f64), torch.randn(1, generator=g, **f64)
    v = {"wo": [Wp, wv], "bo": [bp, bv]}
    H_pi, H_v = torch.randn(M, h, generator=g, **f64), torch.randn(M, h, generator=g, **f64)
    _, act, teach = _rows(M, na, seed=9)
    act[::5] = 1
    Rs, Adv = torch.randn(M, generator=g, **f64), torch.randn(M, generator=g, **f64)
    scale = 1.0 / M
    ref = heads_imit_ref(_Lay([na]), v, 0, H_pi, H_v, act, teach, Rs, Adv, scale, v_coef, beta, lam)
    hp, hv = H_pi.clone().requires_grad_(True), H_v.clone().requires_grad_(True)
    logits = hp @ Wp + bp
    pi = torch.softmax(logits, -1)
    lp = torch.log(pi.clamp(1e-10, 1.0))
    ent = -(pi * lp).sum(-1)
    val = (hv @ wv + bv)[:, 0]
    pl = -(lp.gather(1, act[:, None])[:, 0] * Adv).sum() * scale
    vl = 0.5 * v_coef * ((Rs - val) ** 2).sum() * scale
    el = -beta * ent.sum() * scale
    il, ce = imit_loss(logits, teach, lam, scale)
    dhp, dhv = torch.autograd.grad(pl + vl + el + il, [hp, hv])
    torch.testing.assert_close(ref["dH_pi"], dhp, rtol=1e-10, atol=1e-14)
    torch.testing.assert_close(ref["dH_v"], dhv, rtol=1e-10, atol=1e-14)
    torch.testing.assert_close(ref["stats"], torch.stack([pl, vl, el, ce]).detach(), rtol=1e-12, atol=0)


# ---- configuration --------------------------------------------------------------------------------------------------
def _cfg(agent="ma2c", **mc):
    c = configparser.ConfigParser()
    c.read_string(_ini(agent, 120, 240))
    for k, v in mc.items():
        c["MODEL_CONFIG"][k] = str(v)
    return c


@pytest.mark.parametrize("mc,agent,key", [
    (dict(teacher="pressure", imitation_coef_init=1), "ma2c", "teacher"),
    (dict(teacher="fixedtime", imitation_coef_init=1), "ma2c", "teacher"),
    (dict(teacher="actuated", imitation_coef_init=1), "ia2c", "teacher"),
    (dict(imitation_coef_init=1), "ma2c", "imitation_coef_init"),
    (dict(imitation_decay="linear"), "ia2c", "imitation_decay"),
    (dict(imitation_coef_min=0), "ma2c", "imitation_coef_min"),
    (dict(imitation_ratio=0.5), "ma2c", "imitation_ratio"),
    (dict(teacher="greedy"), "ma2c", "imitation_coef_init"),
    (dict(teacher="greedy", imitation_coef_init=-1), "ma2c", "imitation_coef_init"),
    (dict(teacher="greedy", imitation_coef_init="nan"), "ma2c", "imitation_coef_init"),
    (dict(teacher="greedy", imitation_coef_init="inf"), "ma2c", "imitation_coef_init"),
    (dict(teacher="maxpressure", imitation_coef_init=1, imitation_coef_min=-0.1), "ma2c", "imitation_coef_min"),
    (dict(teacher="maxpressure", imitation_coef_init=1, imitation_decay="exp"), "ma2c", "imitation_decay"),
    (dict(teacher="maxpressure", imitation_coef_init=1, imitation_ratio=0), "ma2c", "imitation_ratio"),
    (dict(teacher="maxpressure", imitation_coef_init=1), "iqll", "teacher"),
    (dict(teacher="maxpressure", imitation_coef_init=1), "iqld", "teacher"),
])
def test_refusals_name_their_key(mc, agent, key):
    from deeprl_signal_control_b200.agents.models import check_imitation
    with pytest.raises(ValueError, match=key):
        check_imitation(_cfg(agent, **mc)["MODEL_CONFIG"], agent)


def test_program_controllers_are_refused_with_the_reason():
    from deeprl_signal_control_b200.agents.learner import check_teacher
    for name in ("fixedtime", "actuated"):
        with pytest.raises(ValueError, match="yellow and all-red"):
            check_teacher(name)
    assert check_teacher(None) is None and check_teacher("greedy") == "greedy"


@pytest.mark.parametrize("entry", ["train", "population", "sweep", "iql_population", "iql_sweep"])
def test_entry_points_refuse_before_any_directory(tmp_path, entry):
    from deeprl_signal_control_b200.agents import train as tr
    agent = "iqll" if entry.startswith("iql") else "ma2c"
    bad = _cfg(agent, teacher="maxpressure", imitation_coef_init=1) if agent == "iqll" else \
        _cfg(agent, imitation_coef_init=1)
    p = tmp_path / "bad.ini"
    with open(p, "w") as f:
        bad.write(f)
    out = tmp_path / "out"
    with pytest.raises(ValueError, match="teacher" if agent == "iqll" else "imitation_coef_init"):
        if entry == "train":
            tr.train(str(p), str(out), n_replicas=64)
        elif entry == "population":
            tr.train(str(p), str(out), n_replicas=64, seeds=[1, 2])
        elif entry == "sweep":
            tr.train_sweep([str(p)], str(out), n_replicas=64)
        elif entry == "iql_population":
            tr.train_iql_population(str(p), str(out), [1, 2], n_replicas=64)
        else:
            tr.train_iql_sweep([str(p)], str(out), n_replicas=64)
    assert not out.exists()


def test_defaults_and_schedule_values():
    from deeprl_signal_control_b200.agents.models import check_imitation, imitation_scheduler
    from deeprl_signal_control_b200.agents.trainer import schedule_values
    c = _cfg(teacher="maxpressure", imitation_coef_init=0.8)["MODEL_CONFIG"]
    assert check_imitation(c, "ma2c") == "maxpressure"
    s = imitation_scheduler(c, 7200)                            # constant by default
    assert [schedule_values(s, 120) for _ in range(3)] == [0.8, 0.8, 0.8]
    # linear from 1 to the default floor 0 over total_step * imitation_ratio = 7200 * 0.25 = 1800 control steps
    c = _cfg(teacher="greedy", imitation_coef_init=1.0, imitation_decay="linear", imitation_ratio=0.25)["MODEL_CONFIG"]
    s = imitation_scheduler(c, 7200)
    got = [schedule_values(s, 120) for _ in range(17)]
    np.testing.assert_allclose(got[:15], [1.0 - 120.0 * (k + 1) / 1800 for k in range(15)], rtol=1e-12, atol=1e-12)
    assert got[14] == pytest.approx(0.0, abs=1e-12) and got[15:] == [0.0, 0.0]
    # with a floor, and imitation_ratio at its default 1
    c = _cfg(teacher="greedy", imitation_coef_init=2.0, imitation_decay="linear", imitation_coef_min=0.5)["MODEL_CONFIG"]
    s = imitation_scheduler(c, 1200)
    got = [schedule_values(s, 120) for _ in range(10)]
    np.testing.assert_allclose(got, [max(0.5, 2.0 * (1 - 120.0 * (k + 1) / 1200)) for k in range(10)], rtol=1e-12)
    assert check_imitation(_cfg()["MODEL_CONFIG"], "ma2c") is None


# ---- sweeps ---------------------------------------------------------------------------------------------------------
def test_sweep_members_may_differ_in_imitation_keys_only():
    from deeprl_signal_control_b200.agents.train import IMITATION_SWEEP_KEYS, SWEEP_CONFIG_KEYS, sweep_members
    keys = dict(SWEEP_CONFIG_KEYS, MODEL_CONFIG=SWEEP_CONFIG_KEYS["MODEL_CONFIG"] + IMITATION_SWEEP_KEYS)
    a = _cfg(teacher="maxpressure", imitation_coef_init=1.0, imitation_decay="linear", imitation_ratio=0.25)
    b = _cfg(teacher="maxpressure", imitation_coef_init=0.5, imitation_decay="constant", imitation_coef_min=0.1,
             imitation_ratio=0.5)
    assert [n for n, _, _ in sweep_members({"a": a, "b": b}, keys)] == ["a", "b"]
    with pytest.raises(ValueError, match="teacher differs"):
        sweep_members({"a": a, "b": _cfg(teacher="greedy", imitation_coef_init=1.0, imitation_decay="linear",
                                         imitation_ratio=0.25)}, keys)
    with pytest.raises(ValueError, match="teacher differs"):
        sweep_members({"a": a, "b": _cfg()}, keys)
    # the plain sweep keys are unchanged: imitation keys differ only where train_sweep allows them
    with pytest.raises(ValueError, match="imitation_coef_init differs"):
        sweep_members({"a": a, "b": b})


def test_train_sweep_checks_every_members_imitation_keys(tmp_path):
    from deeprl_signal_control_b200.agents.train import train_sweep
    paths = []
    for name, lam in (("a", "1.0"), ("b", "-2")):
        p = tmp_path / ("%s.ini" % name)
        with open(p, "w") as f:
            _cfg(teacher="maxpressure", imitation_coef_init=lam).write(f)
        paths.append(str(p))
    with pytest.raises(ValueError, match="imitation_coef_init"):
        train_sweep(paths, str(tmp_path / "out"), n_replicas=64)
    assert not (tmp_path / "out").exists()


# ---- summaries ------------------------------------------------------------------------------------------------------
def test_summary_tags_of_a_five_column_record():
    from deeprl_signal_control_b200.agents.summary import a2c_events, a2c_values
    rec = np.array([[0.5, 0.25, -0.125, 3.0, 1.5], [0.75, 0.5, -0.25, 4.0, 1.25]], np.float32)
    ev = a2c_events("fplstm_0a", rec, 120, 120)
    assert [s for s, _ in ev] == [120, 240]
    for (_, vals), r in zip(ev, rec):
        assert sorted(vals) == sorted(['loss/fplstm_0a_policy_loss', 'loss/fplstm_0a_value_loss',
                                       'loss/fplstm_0a_total_loss', 'train/fplstm_0a_gradnorm',
                                       'loss/fplstm_0a_imitation_loss'])
        assert vals['loss/fplstm_0a_imitation_loss'] == r[4]
        assert vals['loss/fplstm_0a_total_loss'] == np.float32(np.float32(r[0] + r[1]) + r[2])   # without imitation
    assert 'loss/lstm_0a_imitation_loss' not in a2c_values("lstm_0a", rec[0, :4])
