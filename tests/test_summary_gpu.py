"""GPU: the TensorBoard event log of the training driver (`train(..., summaries=True)`) on the grid config of
test_train_driver_gpu.py (R = 16, T = 120, 360 steps, all_test).

* Weights and optimiser state with summaries on against a run without the argument: bit for bit for IQL; for A2C within
  the bound test_train_driver_gpu.py sets for two runs of one build (its weight-gradient kernels add with atomics, so
  two A2C runs differ in the last bits whether summaries are on or not).
* The first update's A2C scalars against oracle/learner_ref.py in float64 (heads_ref on the run's bf16 activation store
  for MA2C, fc_update_ref for the FC policy) within the bound of the update tests (rtol 1e-4); gradnorm is the
  learner's norms[0] bit for bit.
* IQL: loss / gradnorm of the last update's rounds are the learner's losses / norms buffers bit for bit; the first
  round's q / tq match a float64 recomputation from the ring entries at that round's replay indices.
* train_reward equals the training rows of train_reward.csv, test_reward the mean of each test's rows.
* Summaries off leaves log/ with the text log only and issues the launches of a run without the argument.
* Two gloo ranks on one GPU against the one-process run: the same tags and steps, the first update's values within
  1e-6 relative (the ranks sum the same rows in another order, so the last bits differ), and rank 1 writes no file.
"""
import datetime
import os
import socket

import numpy as np
import pytest
import torch

from tests.test_train_driver_gpu import R, _ini, _rows

pytestmark = pytest.mark.gpu
T = 120
AGENTS = [("ma2c", "lstm"), ("ia2c", "fc"), ("iqll", "lstm"), ("iqld", "lstm")]
NAME = {"ma2c": "fplstm_0a", "ia2c": "fc_0a", "iqll": "lr_0a", "iqld": "dqn_0a"}
A2C_TAGS = ["loss/{n}_policy_loss", "loss/{n}_value_loss", "loss/{n}_total_loss", "train/{n}_gradnorm"]
IQL_TAGS = ["train/{n}_loss", "train/{n}_q", "train/{n}_tq", "train/{n}_gradnorm"]
A2C_DRIFT = 1e-6           # test_train_driver_gpu.py: two A2C runs of one build differ by a few 1e-8


class FirstUpdate:
    """Records the inputs and outputs of the first A2C backward / IQL round of a run."""

    def __init__(self):
        from deeprl_signal_control_b200.agents.learner import BatchedA2C
        from deeprl_signal_control_b200.agents.learner_fc import BatchedFcA2C
        from deeprl_signal_control_b200.agents.learner_iql import BatchedIQL
        self.snap = None
        self.saved = [(BatchedA2C, "backward", BatchedA2C.backward), (BatchedFcA2C, "backward", BatchedFcA2C.backward),
                      (BatchedIQL, "td_round", BatchedIQL.td_round)]
        me, orig_td = self, BatchedIQL.td_round

        def wrap_a2c(orig):
            def backward(m, boot, lr, beta):
                first = me.snap is None
                if first:
                    me.snap = dict(P=m.P.clone(), obs=m.obs_hist[:m.T].clone(), beta=beta)
                out = orig(m, boot, lr, beta)
                if first:
                    me.snap.update(Rs=m.Rs.clone(), Adv=m.Adv.clone(), act=m.act_hist.clone(), stats=m.stats.clone(),
                                   norms=m.norms.clone(), st_h=None if m.st_h is None else m.st_h.clone(),
                                   store=bool(m.store_acts))
                return out
            return backward

        def td_round(m, rnd, lr, idx=None, rec=None):
            first = me.snap is None
            if first:
                me.snap = dict(P=m.P.clone(), ring={k: getattr(m, k)[:m.size].clone()
                                                    for k in ("s", "s1", "a", "r", "done")})
            out = orig_td(m, rnd, lr, idx, rec)
            if first:
                me.snap.update(idx=m.idx.clone())
            return out
        BatchedA2C.backward = wrap_a2c(self.saved[0][2])
        BatchedFcA2C.backward = wrap_a2c(self.saved[1][2])
        BatchedIQL.td_round = td_round

    def restore(self):
        for c, name, f in self.saved:
            setattr(c, name, f)


def _train(d, agent, policy, **kw):
    from deeprl_signal_control_b200.agents.train import train
    d.mkdir(parents=True)
    cfg = d / ("config_%s_large.ini" % agent)
    cfg.write_text(_ini(agent, 360, 240))
    base = d / agent
    return base, train(str(cfg), str(base), "all_test", n_replicas=R, policy=policy, **kw)


def _events(base):
    from deeprl_signal_control_b200.agents.summary import event_files, read_records, decode_event
    files = event_files(str(base / "log"))
    assert len(files) == 1, files
    return [decode_event(r) for r in read_records(files[0])[1:]]


def _series(events, tag):
    return [(s, v) for _, s, _, vals in events for k, v in vals if k == tag]


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    """{agent: (on: (base, ns, first update), off: (base, ns))} with the one-process runs of every agent"""
    out = tmp_path_factory.mktemp("summaries")
    res = {}
    for agent, policy in AGENTS:
        rec = FirstUpdate()
        try:
            on = _train(out / "on" / agent, agent, policy, summaries=True)
        finally:
            rec.restore()
        off = _train(out / "off" / agent, agent, policy)
        res[agent] = ((on[0], on[1], rec.snap), off)
    return res


def _state(model):
    if model.name == "iql":
        return {"P": model.P, "M": model.M, "V": model.V}
    return {"P": model.batched.P, "MS": model.batched.MS}


@pytest.mark.parametrize("agent,policy", AGENTS)
def test_summaries_leave_training_unchanged(runs, agent, policy):
    (_, on, _), (_, off) = runs[agent]
    a, b = _state(on.model), _state(off.model)
    if agent.startswith("iq"):
        for k in a:
            assert torch.equal(a[k], b[k]), k
        assert on.model.t == off.model.t > 0
        assert on.trainer.episode_rewards == off.trainer.episode_rewards
    else:
        for k in a:
            assert float((a[k] - b[k]).abs().max()) <= A2C_DRIFT, k
        np.testing.assert_allclose(on.trainer.episode_rewards, off.trainer.episode_rewards, rtol=1e-5)
    assert on.trainer.n_updates == off.trainer.n_updates > 0


@pytest.mark.parametrize("agent,policy", AGENTS)
def test_tags_steps_and_rewards(runs, agent, policy):
    (base, ns, _), _ = runs[agent]
    ev = _events(base)
    n = NAME[agent]
    df = _rows(base)
    train_rows = df[df.test_id == -1]
    assert _series(ev, "train_reward") == [(int(s), float(np.float32(v))) for s, v in
                                           zip(train_rows.step, train_rows.avg_reward)]
    tests = df[df.test_id >= 0].groupby("step").avg_reward.mean()
    assert _series(ev, "test_reward") == [(int(s), float(np.float32(v))) for s, v in tests.items()]
    assert list(tests.index) == [240]
    if agent.startswith("iq"):
        # batch_size 20: an update every 20 steps from step 20 on, rounds at +0 .. +9
        want = [s + k for s in range(20, 361, 20) for k in range(10)]
        tags = [t.format(n=n) for t in IQL_TAGS]
    else:
        want = [120, 240, 360]                                      # batch_size = T
        tags = [t.format(n=n) for t in A2C_TAGS]
    for tag in tags:
        got = _series(ev, tag)
        assert [s for s, _ in got] == want, tag
        assert np.isfinite([v for _, v in got]).all(), tag
    assert sorted({k for _, _, _, vals in ev for k, _ in vals}) == sorted(tags + ["train_reward", "test_reward"])


@pytest.mark.parametrize("agent,policy", [("ma2c", "lstm"), ("ia2c", "fc")])
def test_first_a2c_update_matches_float64(runs, agent, policy):
    from oracle.learner_ref import fc_update_ref, heads_ref
    (base, ns, snap), _ = runs[agent]
    b = ns.model.batched
    lay = b.lay
    scale = 1.0 / (T * R)
    f64 = dict(dtype=torch.float64)
    Rs, Adv, act = (snap[k][:, :, 0].reshape(-1) for k in ("Rs", "Adv", "act"))
    if policy == "lstm":
        assert snap["store"]
        st_h = snap["st_h"]                                        # [chunks = 1][U][T][R][h] bf16: what the kernel reads
        v = lay.views(snap["P"].to(**f64))
        ref = heads_ref(lay, v, 0, st_h[0, 0].reshape(-1, lay.h).to(**f64), st_h[0, 1].reshape(-1, lay.h).to(**f64),
                        act, Rs.to(**f64), Adv.to(**f64), scale, b.v_coef, snap["beta"])["stats"]
    else:
        _, ref = fc_update_ref(lay, snap["P"], snap["obs"], snap["act"], snap["Rs"], snap["Adv"], scale, b.v_coef,
                               snap["beta"], b.chunk, agents=range(0, 1))
    ref = ref.cpu().numpy()
    got = snap["stats"][:3].cpu().numpy()
    np.testing.assert_allclose(got, ref, rtol=1e-4)
    ev = dict((k, v) for _, s, _, vals in _events(base) if s == 120 for k, v in vals)
    n = NAME[agent]
    np.testing.assert_allclose([ev["loss/%s_policy_loss" % n], ev["loss/%s_value_loss" % n]], ref[:2], rtol=1e-4)
    np.testing.assert_allclose(ev["loss/%s_total_loss" % n], ref.sum(), rtol=1e-4, atol=1e-4 * np.abs(ref).sum())
    assert ev["loss/%s_policy_loss" % n] == float(got[0]) and ev["loss/%s_value_loss" % n] == float(got[1])
    assert ev["train/%s_gradnorm" % n] == float(snap["norms"][0])
    print("\n%s first update: policy %.6g value %.6g entropy %.6g (float64 %s), gradnorm %.6g"
          % (agent, *got, ref, float(snap["norms"][0])))


def _q64(P, lay, a, S):
    """Agent a's Q values in float64 from the flat weights (IQL._q)."""
    p = {k: t.to(torch.float64) for k, t in lay.views(P)[a].items()}
    if lay.model_type != "dqn":
        return S @ p["q/w"] + p["q/b"]
    n_w = int(lay.n_w[a])
    if n_w == 0:
        h = torch.relu(S @ p["q_fcw/w"] + p["q_fcw/b"])
    else:
        n_s = S.shape[1] - n_w
        h = torch.cat([torch.relu(S[:, :n_s] @ p["q_fcw/w"] + p["q_fcw/b"]),
                       torch.relu(S[:, n_s:] @ p["q_fct/w"] + p["q_fct/b"])], 1)
    h = torch.relu(h @ p["q_fc_0/w"] + p["q_fc_0/b"])
    return h @ p["q/w"] + p["q/b"]


@pytest.mark.parametrize("agent", ["iqll", "iqld"])
def test_iql_scalars(runs, agent):
    (base, ns, snap), _ = runs[agent]
    m = ns.model
    ev = _events(base)
    n = NAME[agent]
    # the last update's rounds are what the learner's losses / norms buffers hold
    loss, norm = _series(ev, "train/%s_loss" % n)[-10:], _series(ev, "train/%s_gradnorm" % n)[-10:]
    assert [v for _, v in loss] == [float(x) for x in m.losses[:, 0].cpu()]
    assert [v for _, v in norm] == [float(x) for x in m.norms[:, 0].cpu()]
    # the first round's q / tq from the ring entries at its replay indices
    ring, idx = snap["ring"], snap["idx"][0].long()                 # agent 0: [R][batch]
    lay = m.lay
    o0, ns0 = int(lay.obs_off[0]), int(lay.n_s[0])
    rr = torch.arange(R, device=idx.device)[:, None].expand_as(idx)
    S = ring["s"][idx, rr, o0:o0 + ns0].reshape(-1, ns0).double()
    S1 = ring["s1"][idx, rr, o0:o0 + ns0].reshape(-1, ns0).double()
    a = ring["a"][idx, rr, 0].reshape(-1).long()
    r = ring["r"][idx, rr, 0].reshape(-1).double()
    done = ring["done"][idx, rr].reshape(-1).bool()
    q0 = _q64(snap["P"], lay, 0, S).gather(1, a[:, None])[:, 0]
    tq = torch.where(done, r, r + m.gamma * _q64(snap["P"], lay, 0, S1).max(1)[0])
    first = {k: _series(ev, "train/%s_%s" % (n, k))[0] for k in ("loss", "q", "tq")}
    assert first["q"][0] == first["tq"][0] == first["loss"][0] == 20
    np.testing.assert_allclose(first["q"][1], float(q0.mean()), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(first["tq"][1], float(tq.mean()), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(first["loss"][1], float(((q0 - tq) ** 2).mean()), rtol=1e-4)


def test_summaries_off_writes_and_launches_nothing(runs, tmp_path):
    (_, on, _), (base_off, off) = runs["ma2c"]
    logs = os.listdir(base_off / "log")
    assert len(logs) == 1 and logs[0].endswith(".log")
    base, explicit = _train(tmp_path / "explicit", "ma2c", "lstm", summaries=False)
    assert len(os.listdir(base / "log")) == 1 and os.listdir(base / "log")[0].endswith(".log")
    assert explicit.model.batched.kernel_launches == off.model.batched.kernel_launches == \
        on.model.batched.kernel_launches > 0
    assert off.trainer.summary_rec is None and explicit.trainer.summary_rec is None


# ---- two gloo ranks on one GPU -------------------------------------------------------------------------------------
WORLD = 2
RANK_AGENTS = [("ma2c", "lstm"), ("iqld", "lstm")]


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=WORLD, timeout=datetime.timedelta(seconds=300))
    from deeprl_signal_control_b200.agents.train import train
    for agent, policy in RANK_AGENTS:
        cfg = os.path.join(out, agent, "config_%s_large.ini" % agent)
        train(cfg, os.path.join(out, agent, agent), "all_test", n_replicas=R, policy=policy, device=0,
              process_group=dist.group.WORLD, summaries=True)
    dist.destroy_process_group()


@pytest.fixture(scope="module")
def world2(tmp_path_factory):
    import torch.multiprocessing as mp
    out = tmp_path_factory.mktemp("summaries_world2")
    for agent, _ in RANK_AGENTS:
        (out / agent).mkdir()
        (out / agent / ("config_%s_large.ini" % agent)).write_text(_ini(agent, 360, 240))
    mp.spawn(_worker, args=(_free_port(), str(out)), nprocs=WORLD, join=True)
    return {agent: out / agent / agent for agent, _ in RANK_AGENTS}


@pytest.mark.parametrize("agent,policy", RANK_AGENTS)
def test_two_ranks_write_the_one_process_log(world2, runs, agent, policy):
    base2 = world2[agent]
    (base1, _, _), _ = runs[agent]
    logs = os.listdir(base2 / "log")                               # rank 0's text log and event file, nothing else
    assert len(logs) == 2 and sorted(f.startswith("events.out.tfevents.") for f in logs) == [False, True]
    assert [f for f in logs if f.endswith(".log")] and len(os.listdir(base1 / "log")) == 2
    e2, e1 = _events(base2), _events(base1)
    assert [(s, [k for k, _ in vals]) for _, s, _, vals in e2] == [(s, [k for k, _ in vals]) for _, s, _, vals in e1]
    # the first update (A2C: step 120, the end of the first episode set; IQL: its first round) plays the same rows
    first2, first1 = dict(e2[0][3]), dict(e1[0][3])
    assert e2[0][1] == e1[0][1] == (120 if agent == "ma2c" else 20)
    for k in first1:
        assert abs(first2[k] - first1[k]) <= 1e-6 * abs(first1[k]), (k, first2[k], first1[k])
    for _, _, _, vals in e2:
        assert np.isfinite([v for _, v in vals]).all()
