"""CPU: the IQL layouts of tests/iql_layout_envelope.py — the flat Q layout against IQL's own tensors, the float64 round
restatement q_td_ref (tests/test_iql_batched_cpu.py) against IQL.td_update run in float64 (loss, gradient norm, clip and
Adam), the kernels' shared-memory restatement, and planted defects that the GPU bounds must catch."""
import numpy as np
import pytest
import torch

from tests.iql_layout_envelope import (BEYOND, DEFECTS, EDGES, FC32_NO_WAIT, SCENARIOS, agent_batch, moved,
                                       scenario_case, synthetic_case)
from tests.test_iql_batched_cpu import q_td_ref

CASES = ["%s/%s" % c for c in SCENARIOS] + list(EDGES)


def _case(name, tmp_path):
    if name in EDGES:
        return synthetic_case(**EDGES[name])
    return scenario_case(*name.split("/"), str(tmp_path))


def _perturbed(m, seed):
    """IQL weights off the initialisation, biases away from zero"""
    g = torch.Generator().manual_seed(seed)
    for p in m.nets:
        for v in p.values():
            v.data.add_(torch.randn(v.shape, generator=g) * 0.05)
    return m


def _rows(case, n, rng):
    obs = rng.random((n, case.n_obs)) * 2
    obs1 = rng.random((n, case.n_obs)) * 2
    acts = np.stack([rng.integers(0, na, n) for na in case.n_a], 1)
    return obs, obs1, acts, rng.standard_normal((n, len(case.n_a))), rng.random(n) < 0.3


@pytest.mark.parametrize("name", CASES)
def test_qlayout_matches_iql(name, tmp_path):
    c = _case(name, tmp_path)
    m = _perturbed(c.iql(seed=2), 3)
    lay = c.layout(m)
    assert lay.A == len(c.n_s) and lay.max_na == c.max_na and lay.n_obs == c.n_obs
    for i, p in enumerate(m.nets):
        assert list(lay.shapes[i]) == list(p) and all(tuple(v.shape) == lay.shapes[i][k] for k, v in p.items()), i
    flat = lay.pack(m.nets)
    assert flat.shape == (lay.n_params,) and lay.n_params == sum(v.numel() for p in m.nets for v in p.values())
    for i, v in enumerate(lay.views(flat)):
        for k, t in v.items():
            assert torch.equal(t, m.nets[i][k].detach()), (i, k)
    assert torch.equal(lay.pack(lay.views(flat)), flat)
    if c.kind == "dqn":
        assert (lay.n_fc, lay.n_h) == (c.num_fc, c.num_h)
        assert lay.n_ft == (c.num_fc // 4 if any(c.n_w) else 0)
        # every agent block starts at its first tensor and the blocks tile the vector (the clip + Adam ranges)
        starts = list(lay.off_fcw_w) + [lay.n_params]
        assert all(starts[i] < starts[i + 1] for i in range(lay.A)) and starts[0] == 0


def test_smem_restatement_at_the_reference_widths(tmp_path):
    """QLayout.smem_bytes on the grid and Monaco DeepQ layouts, and the TD limit of a wave block next to 6 wait inputs"""
    assert scenario_case("large_grid", "iqld").layout().smem_bytes() == (132832, 194304)
    assert scenario_case("real_net", "iqld").layout().smem_bytes() == (116544, 170848)
    optin = 232448                                     # H100 opt-in shared memory per block
    fit = synthetic_case(**EDGES["td_wave_max"]).layout().smem_bytes()
    over = synthetic_case(**BEYOND["td_wave_beyond"][0]).layout().smem_bytes()
    assert fit[1] <= optin < over[1] and over[0] <= optin


def _iql64(m):
    """the IQL's weights and Adam state as float64 leaves"""
    for i, p in enumerate(m.nets):
        for k in list(p):
            p[k] = p[k].detach().double().requires_grad_(True)
        m.adam[i] = dict(t=0, m={k: torch.zeros_like(v) for k, v in p.items()},
                         v={k: torch.zeros_like(v) for k, v in p.items()})


class _Float64Numpy:
    """numpy whose float32 is float64: IQL.td_update's own statements (np.asarray(x, np.float32)) in float64"""

    def __getattr__(self, k):
        return np.float64 if k == "float32" else getattr(np, k)


@pytest.mark.parametrize("name", CASES)
def test_q_td_ref_equals_td_update_in_float64(name, tmp_path, monkeypatch):
    """two rounds per agent; the clip is on for even agents and off for odd ones"""
    from deeprl_signal_control_b200.agents import models
    c = _case(name, tmp_path)
    m = _perturbed(c.iql(seed=4, total_step=1000), 5)
    lay = c.layout(m)
    _iql64(m)
    monkeypatch.setattr(models, "np", _Float64Numpy())
    rng = np.random.default_rng(6)
    lr = 1e-3
    for i in range(lay.A):
        w = {k: v.detach().numpy().copy() for k, v in m.nets[i].items()}
        adam = dict(t=0, m={k: 0 * v for k, v in w.items()}, v={k: 0 * v for k, v in w.items()})
        n_w = int(lay.n_w[i])
        for rnd in range(2):
            obs, obs1, acts, rw, d = _rows(c, 30, rng)
            o = slice(int(lay.obs_off[i]), int(lay.obs_off[i]) + int(lay.n_s[i]))
            S, S1, A, Rw = obs[:, o], obs1[:, o], acts[:, i], rw[:, i]
            norm = q_td_ref(w, c.kind, n_w, S, A, S1, Rw, d, 0.99)["norm"]
            m.max_grad_norm = norm * (0.5 if i % 2 == 0 else 2.0)
            ref = q_td_ref(w, c.kind, n_w, S, A, S1, Rw, d, 0.99, max_norm=m.max_grad_norm, adam=adam, lr=lr)
            loss, norm = m.td_update(i, S, A, S1, d, Rw, lr)
            assert abs(loss - ref["loss"]) <= 1e-10 * abs(ref["loss"]), (i, rnd)
            assert abs(norm - ref["norm"]) <= 1e-10 * ref["norm"], (i, rnd)
            st = m.adam[i]
            assert st["t"] == ref["adam"]["t"] == rnd + 1
            for k in w:
                for got, want in ((m.nets[i][k].detach().numpy(), ref["w"][k]), (st["m"][k].numpy(), ref["adam"]["m"][k]),
                                  (st["v"][k].numpy(), ref["adam"]["v"][k])):
                    assert np.abs(got - want).max() <= 1e-10 * max(np.abs(want).max(), 1e-30), (i, rnd, k)
            w, adam = ref["w"], ref["adam"]


@pytest.mark.parametrize("name", CASES)
def test_planted_defects_move_the_round_beyond_the_gpu_bounds(name, tmp_path):
    c = _case(name, tmp_path)
    m = _perturbed(c.iql(seed=7), 8)
    lay = c.layout(m)
    P = lay.pack([{k: v.detach().numpy() for k, v in p.items()} for p in m.nets]).astype(np.float64)
    obs, obs1, acts, rw, d = _rows(c, 40, np.random.default_rng(9))
    hits = {}
    for i in range(lay.A):
        w, n_w, S, S1, _ = agent_batch(lay, P, i, obs, obs1)
        base = q_td_ref(w, c.kind, n_w, S, acts[:, i], S1, rw[:, i], d, 0.99)
        for name_d in DEFECTS:
            b = agent_batch(lay, P, i, obs, obs1, name_d)
            if b is None:
                continue
            bad = q_td_ref(b[0], c.kind, b[1], b[2], acts[:, i], b[3], rw[:, i], d, 0.99, mutate=b[4])
            ratio, what = moved(base, bad, c.kind)
            assert ratio >= 10, (i, name_d, what, ratio)
            hits[name_d] = min(hits.get(name_d, np.inf), ratio)
    assert "done mask dropped" in hits and "next agent's observation slice" in hits
    if c.kind == "dqn" and any(c.n_w):
        assert "wait block read as wave inputs" in hits
    if c.kind == "dqn" and any(c.n_w) and not all(c.n_w[:-1]):
        assert "q_fct branch on an agent without a wait block" in hits


def test_beyond_layouts_build_on_the_host():
    """the layouts one past a limit are ordinary IQL models and QLayouts: the refusal is the kernels' (GPU test)"""
    for name, (kw, _) in BEYOND.items():
        c = synthetic_case(**kw)
        lay = c.layout()
        assert lay.n_params == sum(v.numel() for p in c.iql().nets for v in p.values()), name
    assert synthetic_case(**FC32_NO_WAIT).layout().n_ft == 0
