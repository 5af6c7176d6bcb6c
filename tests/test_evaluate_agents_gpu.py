"""GPU: evaluating several agents in one process (agents/evaluator.py:GroupEvaluator, scripts/evaluate_agents.py).

* tscl_policy_step_pi_g against one tscl_policy_step_pi per member slice (seed seeds[k], replica0 0): pi, c, h and act
  bit-identical for ragged members S = (1, 10, 63, 64, 65, 130), act_mode 0 and 1, done 1 then 0, at grid MA2C (dx 224),
  grid IA2C (160), Monaco MA2C (192) and Monaco IA2C (128).
* tscl_q_step_g against one tscl_q_step per member slice: q, act and the bad flag bit-identical for LR and DQN, grid and
  Monaco, mode 0 and 1; a planted out-of-range row of one member is reported in that member's flag with its own key.
* End to end: a base directory with greedy, ia2c, ma2c, iqll, iqld, two ma2c seed members and two ma2c coop_gamma members
  (short episodes, the reference's widths): every entry's three CSVs and <agent>_summary.json are byte-identical to
  scripts/evaluate.py on that directory alone, for the policy types default, deterministic and stochastic.
* Two iqld directories of different widths (num_fc / num_h) on one simulator, one Q launch per layout: each entry's
  CSVs and summary byte-identical to scripts/evaluate.py on that directory alone.
"""
import configparser
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

from tests.test_evaluator_iql_gpu import _iql, _net

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (1, 10, 63, 64, 65, 130)
MEMBER_SEEDS = (12, 13, (1 << 40) + 7, 99, 2 ** 63 + 5, 4)


def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rows(sizes):
    return torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device="cuda")


def _seeds(seeds):
    return torch.tensor(np.array(seeds, dtype=np.uint64).view(np.int64), device="cuda")


@pytest.mark.parametrize("scenario,agent,dx", [("large_grid", "ma2c", 224), ("large_grid", "ia2c", 160),
                                               ("real_net", "ma2c", 192), ("real_net", "ia2c", 128)])
def test_grouped_pi_forward_equals_member_launches(scenario, agent, dx):
    from bench import build_scenario, make_layout
    from deeprl_signal_control_b200 import _lib
    from deeprl_signal_control_b200.agents.learner import BatchedA2C

    class A:
        policy = "lstm"
    A.scenario, A.agent = scenario, agent
    lay = make_layout(build_scenario(A)[0], A)
    assert lay.dx == dx
    lib, K, R = _lib.lib(), len(SIZES), sum(SIZES)
    g = torch.Generator(device="cuda").manual_seed(7)
    ms = []
    for k in range(K):
        m = BatchedA2C(lay, 64, n_step=2, seed=5 + k, chunk=64, store_acts=False)
        m.P.add_(torch.randn(m.P.shape, device="cuda", generator=g) * 0.02)
        m.pack_weights()
        ms.append(m)
    P = torch.stack([m.P for m in ms]).contiguous()
    Wp = torch.stack([m.Wp for m in ms]).contiguous()
    rows, seeds, r0 = _rows(SIZES), _seeds(MEMBER_SEEDS), np.concatenate([[0], np.cumsum(SIZES)])
    c = torch.randn(lay.A, R, lay.h, device="cuda", generator=g)
    h = torch.rand(lay.A, R, lay.h, device="cuda", generator=g) * 2 - 1
    for mode in (0, 1):
        cs, hs = c.clone(), h.clone()
        for step, done in enumerate([1, 0]):
            obs = torch.rand(R, lay.n_obs, device="cuda", generator=g) * 2
            cg, hg = torch.full_like(cs, float("nan")), torch.full_like(hs, float("nan"))
            pig = torch.full((R, lay.A, lay.max_na), float("nan"), device="cuda")
            actg = torch.full((R, lay.A), -1, dtype=torch.int32, device="cuda")
            _lib.check(lib.tscl_policy_step_pi_g(
                ms[0]._h, _p(P), C.c_int64(P.shape[1]), _p(Wp), C.c_int64(Wp[0].numel()), _p(obs), C.c_int32(K), _p(rows),
                C.c_int64(R), _p(cs), _p(hs), _p(cg), _p(hg), _p(pig), _p(actg), C.c_int32(mode), C.c_int32(done),
                _p(seeds), C.c_int64(step), _st()))
            for k, m in enumerate(ms):
                a, b, S = int(r0[k]), int(r0[k + 1]), SIZES[k]
                ck, hk = cs[:, a:b].contiguous(), hs[:, a:b].contiguous()
                c1, h1 = torch.empty_like(ck), torch.empty_like(hk)
                pi1 = torch.empty(S, lay.A, lay.max_na, device="cuda")
                act1 = torch.empty(S, lay.A, dtype=torch.int32, device="cuda")
                _lib.check(lib.tscl_policy_step_pi(
                    m._h, _p(m.P), _p(m.Wp), _p(obs[a:b]), C.c_int64(S), _p(ck), _p(hk), _p(c1), _p(h1), _p(pi1),
                    _p(act1), C.c_int32(mode), C.c_int32(done), C.c_uint64(MEMBER_SEEDS[k]), C.c_int64(step),
                    C.c_int64(0), C.c_int64(0), C.c_int64(0), _st()))
                torch.cuda.synchronize()
                what = (scenario, agent, mode, step, k)
                assert torch.equal(pig[a:b], pi1), what
                assert torch.equal(cg[:, a:b], c1) and torch.equal(hg[:, a:b], h1), what
                assert torch.equal(actg[a:b], act1), what
            cs, hs = cg, hg


class _QMembers:
    def __init__(self, scenario, kind, sizes, positive=False):
        from deeprl_signal_control_b200 import _lib
        from deeprl_signal_control_b200.agents.layout import QLayout
        self.lib, self.check = _lib.lib(), _lib.check
        self.net = _net(scenario, "iqll" if kind == "lr" else "iqld")
        self.ms = [_iql(self.net, kind, seed=3 + k) for k in range(len(sizes))]
        if positive:                    # q well above 0 everywhere: every row's normalised q is a distribution
            for m in self.ms:
                for i, p in enumerate(m.nets):
                    for key, v in p.items():
                        if key.endswith("/b") and v.numel() == int(self.net.n_a_ls[i]):
                            v.data.add_(50.0)
        self.lay = QLayout.from_iql(self.ms[0], self.net.node_obs_off, self.net.n_obs, max_na=self.net.max_na)
        self.h = C.c_void_p()
        self.check(self.lib.tscl_q_create(C.byref(self.lay.as_c()), C.c_int32(0), C.byref(self.h)))
        self.P = torch.stack([self.lay.pack(m.nets).cuda() for m in self.ms]).contiguous()
        self.sizes = sizes

    def close(self):
        self.lib.tscl_q_destroy(self.h)


@pytest.mark.parametrize("scenario", ["large_grid", "real_net"])
@pytest.mark.parametrize("kind", ["lr", "dqn"])
@pytest.mark.parametrize("mode", [0, 1])
def test_grouped_q_forward_equals_member_launches(scenario, kind, mode):
    qm = _QMembers(scenario, kind, SIZES)
    L, K, R = qm.lay, len(SIZES), sum(SIZES)
    r0 = np.concatenate([[0], np.cumsum(SIZES)])
    rows, seeds = _rows(SIZES), _seeds(MEMBER_SEEDS)     # held: the launch reads them after this line
    g = torch.Generator(device="cuda").manual_seed(2)
    try:
        for step in (0, 5):
            obs = torch.rand(R, L.n_obs, device="cuda", generator=g) * 2
            q = torch.full((R, L.A, L.max_na), float("nan"), device="cuda")
            act = torch.full((R, L.A), -1, dtype=torch.int32, device="cuda")
            bad = torch.full((K,), -1, dtype=torch.int64, device="cuda")
            qm.check(qm.lib.tscl_q_step_g(qm.h, _p(qm.P), C.c_int64(L.n_params), _p(obs), C.c_int32(K), _p(rows),
                                          C.c_int64(R), _p(q), _p(act), C.c_int32(mode), _p(seeds), C.c_int64(step),
                                          _p(bad), _st()))
            for k in range(K):
                a, b, S = int(r0[k]), int(r0[k + 1]), SIZES[k]
                q1 = torch.empty(S, L.A, L.max_na, device="cuda")
                a1 = torch.empty(S, L.A, dtype=torch.int32, device="cuda")
                b1 = torch.full((1,), -1, dtype=torch.int64, device="cuda")
                qm.check(qm.lib.tscl_q_step(qm.h, _p(qm.P[k]), _p(obs[a:b]), C.c_int64(S), _p(q1), _p(a1),
                                            C.c_int32(mode), C.c_uint64(MEMBER_SEEDS[k]), C.c_int64(step), C.c_int64(0),
                                            _p(b1), _st()))
                torch.cuda.synchronize()
                assert torch.equal(q[a:b], q1) and torch.equal(act[a:b], a1), (step, k)
                assert int(bad[k]) == int(b1[0]), (step, k)
    finally:
        qm.close()


@pytest.mark.parametrize("kind", ["lr", "dqn"])
def test_grouped_q_reports_a_planted_row_with_its_members_key(kind):
    qm = _QMembers("large_grid", kind, SIZES, positive=True)
    L, K, R = qm.lay, len(SIZES), sum(SIZES)
    r0 = np.concatenate([[0], np.cumsum(SIZES)])
    member, local, agent, step = 4, 7, 3, 9
    a, b, o = int(r0[member]), int(r0[member + 1]), int(L.obs_off[agent])
    want = [-1] * K
    want[member] = (local << 40) | (step << 16) | agent
    try:
        obs = torch.rand(R, L.n_obs, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
        # the planted row: observations far outside their range, the first value whose q is not a distribution in the
        # member's own launch (both signs, or not finite; a NaN alone would not do for DQN, whose relu maps it to 0)
        for v in (1e4, -1e4, 1e30, -1e30, float("inf"), float("-inf")):
            obs[a + local, o:o + int(L.n_s[agent])] = v
            q1 = torch.empty(b - a, L.A, L.max_na, device="cuda")
            a1 = torch.empty(b - a, L.A, dtype=torch.int32, device="cuda")
            b1 = torch.full((1,), -1, dtype=torch.int64, device="cuda")
            qm.check(qm.lib.tscl_q_step(qm.h, _p(qm.P[member]), _p(obs[a:b]), C.c_int64(b - a), _p(q1), _p(a1),
                                        C.c_int32(1), C.c_uint64(MEMBER_SEEDS[member]), C.c_int64(step), C.c_int64(0),
                                        _p(b1), _st()))
            if int(b1[0]) == want[member]:
                break
        assert int(b1[0]) == want[member]
        q = torch.zeros(R, L.A, L.max_na, device="cuda")
        act = torch.zeros(R, L.A, dtype=torch.int32, device="cuda")
        bad = torch.full((K,), -1, dtype=torch.int64, device="cuda")
        rows, seeds = _rows(SIZES), _seeds(MEMBER_SEEDS)
        qm.check(qm.lib.tscl_q_step_g(qm.h, _p(qm.P), C.c_int64(L.n_params), _p(obs), C.c_int32(K), _p(rows),
                                      C.c_int64(R), _p(q), _p(act), C.c_int32(1), _p(seeds), C.c_int64(step), _p(bad),
                                      _st()))
        torch.cuda.synchronize()
        assert bad.cpu().tolist() == want
        assert int(act[a + local, agent]) == 0
    finally:
        qm.close()


# ---- end to end -------------------------------------------------------------------------------------------------------
SEEDS = [10000, 20000, 30000]
EPISODE_SEC = 60
# (entry, [ENV_CONFIG] changes, weight seed)
ENTRIES = [("greedy", {}, 0), ("ia2c", {}, 1), ("ma2c", {}, 2), ("iqll", {}, 3), ("iqld", {}, 4),
           ("seed13/ma2c", {"seed": "13"}, 5), ("seed14/ma2c", {"seed": "14"}, 6),
           ("cg075/ma2c", {"coop_gamma": "0.75"}, 7), ("cg050/ma2c", {"coop_gamma": "0.5"}, 8)]


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "scripts", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _make_base(base, entries):
    from tests.test_train_driver_gpu import A2C_MODEL, GRID, IQL_MODEL, TRAIN
    from deeprl_signal_control_b200.envs import make_env
    from deeprl_signal_control_b200.agents.models import IA2C, IQL, MA2C
    for entry, changes, wseed in entries:
        agent = os.path.basename(entry)
        model = A2C_MODEL if agent in ("ia2c", "ma2c", "greedy") else IQL_MODEL
        c = configparser.ConfigParser()
        c.read_string(model + TRAIN % (120, 120) + GRID % (agent, ",".join(map(str, SEEDS))))
        c["ENV_CONFIG"]["episode_length_sec"] = str(EPISODE_SEC)
        for k, v in changes.items():                    # a [MODEL_CONFIG] key where it names one, else [ENV_CONFIG]
            c["MODEL_CONFIG" if k in c["MODEL_CONFIG"] else "ENV_CONFIG"][k] = v
        d = os.path.join(base, entry)
        for sub in ("data", "model"):
            os.makedirs(os.path.join(d, sub))
        with open(os.path.join(d, "data", "config.ini"), "w") as f:
            c.write(f)
        if agent == "greedy":
            continue
        env = make_env(c["ENV_CONFIG"], len(SEEDS), d + "/", is_record=False)
        mc = c["MODEL_CONFIG"]
        kw = dict(n_replicas=1, obs_off=env._tables.node_obs_off, seed=wseed)
        if agent == "ma2c":
            m = MA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, env.n_f_ls, 0, mc, **kw)
        elif agent == "ia2c":
            m = IA2C(env.n_s_ls, env.n_a_ls, env.n_w_ls, 0, mc, **kw)
        else:
            m = IQL(env.n_s_ls, env.n_a_ls, env.n_w_ls, 0, mc, seed=wseed, model_type="dqn" if agent == "iqld" else "lr")
            for i, p in enumerate(m.nets):      # q well above 0: the stochastic policy's normalised q is a distribution
                for key, v in p.items():
                    if key.endswith("/b") and v.numel() == int(env.n_a_ls[i]):
                        v.data.add_(50.0)
        m.save(os.path.join(d, "model"), 120)


def _bytes(path):
    with open(path, "rb") as f:
        return f.read()


def _evaluate_against_solo(tmp_path, entries, policy_type):
    """evaluate_agents.py on `entries`, then evaluate.py on each directory alone: the same bytes in every output."""
    base = str(tmp_path / "B")
    _make_base(base, entries)
    seeds = ",".join(map(str, SEEDS))
    out = _load("evaluate_agents").main(["--base-dir", base, "--agents", ",".join(e for e, _, _ in entries),
                                         "--evaluation-policy-type", policy_type, "--evaluation-seeds", seeds])
    assert [lab for lab, _ in out] == [e for e, _, _ in entries]
    solo = _load("evaluate")
    for entry, _, _ in entries:
        agent = os.path.basename(entry)
        x = str(tmp_path / "solo" / entry)
        solo.main(["--agent-dir", os.path.join(base, entry), "--output-dir", x, "--evaluation-seeds", seeds,
                   "--evaluation-policy-type", policy_type])
        got_dir = os.path.join(base, "eva_data", os.path.dirname(entry))
        names = ["large_grid_%s_%s.csv" % (agent, w) for w in ("control", "traffic", "trip")] + ["%s_summary.json" % agent]
        for n in names:
            assert _bytes(os.path.join(got_dir, n)) == _bytes(os.path.join(x, n)), (entry, n)
    rows = open(os.path.join(base, "eva_data", "summary.csv")).read().splitlines()
    assert len(rows) == 1 + len(entries) and rows[0].startswith("entry,mean_reward")
    assert os.listdir(os.path.join(base, "eva_log"))


@pytest.mark.parametrize("policy_type", ["default", "deterministic", "stochastic"])
def test_evaluate_agents_equals_one_directory_at_a_time(tmp_path, policy_type):
    _evaluate_against_solo(tmp_path, ENTRIES, policy_type)


def test_iql_entries_of_two_layouts_equal_one_directory_at_a_time(tmp_path):
    """Two iqld directories that share a simulator but not a Q layout: each layout has its own grouped launch."""
    _evaluate_against_solo(tmp_path, [("w128/iqld", {}, 3), ("w64/iqld", {"num_fc": "64", "num_h": "32"}, 4)], "default")
