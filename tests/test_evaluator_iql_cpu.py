"""CPU: the pieces of batched IQL evaluation that need no GPU — a float64 restatement of the LRQPolicy / DeepQPolicy
forward (agents/policies.py:341-389) against the reference graph's own q-values (tests/golden/learner_iql.npz), the
flat Q parameter layout (agents/layout.py:QLayout) against IQL.nets and IQL checkpoints, the Monaco tables of the IQL
agents, and the agent-name -> model-type map of scripts/evaluate.py (main.py:179-190)."""
import configparser
import gzip
import os
import shutil
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
INI = """
[MODEL_CONFIG]
gamma = 0.99
lr_init = 1e-4
lr_decay = constant
epsilon_init = 1.0
epsilon_min = 0.01
epsilon_decay = linear
epsilon_ratio = 0.5
max_grad_norm = 40
batch_size = 20
buffer_size = 1000
reward_norm = 1.0
reward_clip = 2.0
num_fc = 128
num_h = 64
"""


def q_forward_ref(model_type, w, S, n_w=0, with_scale=False):
    """float64 q-values of one agent: w = {name: array} with the IQL / TF names (q/w, q_fcw/b, ...), S [M][n_s].
    with_scale: also the row scale of an fp32 evaluation, max_j (|b_j| + sum_k |x_k W_kj|) over the output layer's terms
    (x = S for lr, the last hidden layer for dqn)."""
    f = lambda k: np.asarray(w[k], np.float64)
    S = np.asarray(S, np.float64)
    out = lambda x: ((x @ f("q/w") + f("q/b"), (np.abs(x) @ np.abs(f("q/w")) + np.abs(f("q/b"))).max(1))
                     if with_scale else x @ f("q/w") + f("q/b"))
    if model_type == "lr":
        return out(S)
    n = S.shape[1] - n_w
    h = np.maximum(S[:, :n] @ f("q_fcw/w") + f("q_fcw/b"), 0.0)
    if n_w > 0:
        h = np.concatenate([h, np.maximum(S[:, n:] @ f("q_fct/w") + f("q_fct/b"), 0.0)], 1)
    h = np.maximum(h @ f("q_fc_0/w") + f("q_fc_0/b"), 0.0)
    return out(h)


def model_config():
    cp = configparser.ConfigParser()
    cp.read_string(INI)
    return cp["MODEL_CONFIG"]


@pytest.mark.parametrize("kind", ["lr", "dqn"])
def test_float64_q_forward_equals_the_reference_graph(kind):
    z = np.load(os.path.join(GOLD, "learner_iql.npz"))
    checked = 0
    for k in range(3):
        for i in range(2):
            pre = "%s/k%d/a%d" % (kind, k, i)
            wp = "%s/w%d/%s_%da_q/" % (kind, k, kind, i)
            w = {n[len(wp):]: z[n] for n in z.files if n.startswith(wp)}
            got = q_forward_ref(kind, w, z[pre + "/obs"])
            want = z[pre + "/q"]
            assert got.shape == want.shape
            np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-6 * float(np.abs(want).max()))
            checked += 1
    assert checked == 6


def _iql(kind, n_s, n_a, n_w, seed=0):
    from deeprl_signal_control_b200.agents.models import IQL
    m = IQL(n_s, n_a, n_w, 0, model_config(), seed=seed, model_type=kind, device="cpu")
    g = torch.Generator().manual_seed(seed + 7)
    for p in m.nets:
        for v in p.values():
            v.data.add_(torch.randn(v.shape, generator=g) * 0.1)        # biases away from zero, weights off the init
    return m


CASES = [("lr", [24, 30, 36], [5, 3, 4], [6, 6, 6]), ("dqn", [24, 30, 36], [5, 3, 4], [6, 6, 6]),
         ("dqn", [5, 17, 34, 9], [2, 6, 3, 4], [0, 0, 0, 0]), ("dqn", [12, 20, 8], [3, 2, 4], [4, 0, 2])]


@pytest.mark.parametrize("kind,n_s,n_a,n_w", CASES)
def test_qlayout_packs_iql_nets_and_checkpoints(kind, n_s, n_a, n_w, tmp_path):
    from deeprl_signal_control_b200.agents.layout import QLayout
    m = _iql(kind, n_s, n_a, n_w)
    off = np.concatenate([[0], np.cumsum(n_s)])
    lay = QLayout.from_iql(m, off, int(off[-1]) + 3, max_na=8)
    assert (lay.n_fc, lay.n_ft, lay.n_h) == ((128, 32 if any(n_w) else 0, 64) if kind == "dqn" else (0, 0, 0))
    flat = lay.pack(m.nets)
    assert flat.dtype == torch.float32 and flat.shape == (lay.n_params,)
    assert lay.n_params == sum(v.numel() for p in m.nets for v in p.values())
    views = lay.views(flat)
    for i, p in enumerate(m.nets):
        assert set(views[i]) == set(p)
        for k, v in p.items():
            assert torch.equal(views[i][k], v.detach()), (i, k)
    # the offsets the kernel reads address the same floats
    for i, p in enumerate(m.nets):
        for k, v in p.items():
            o = int(getattr(lay, QLayout.OFF[k])[i])
            assert torch.equal(flat[o:o + v.numel()], v.detach().reshape(-1)), (i, k)
    # numpy nets pack to the same vector
    np.testing.assert_array_equal(lay.pack([{k: v.detach().numpy() for k, v in p.items()} for p in m.nets]), flat.numpy())
    # save -> load into a differently initialised IQL -> the same packed vector
    m.save(str(tmp_path) + "/", 300)
    m2 = _iql(kind, n_s, n_a, n_w, seed=5)
    assert not torch.equal(lay.pack(m2.nets), flat)
    assert m2.load(str(tmp_path) + "/") is True
    assert torch.equal(QLayout.from_iql(m2, off, int(off[-1]) + 3, max_na=8).pack(m2.nets), flat)
    # the C image
    c = lay.as_c()
    assert c.n_agents == len(n_s) and c.model == (1 if kind == "dqn" else 0) and c.n_params == lay.n_params
    assert [c.off_q_w[i] for i in range(len(n_s))] == [int(x) for x in lay.off_q_w]


def test_qlayout_rejects_a_model_of_other_widths():
    from deeprl_signal_control_b200.agents.layout import QLayout
    m = _iql("dqn", [12, 20], [3, 2], [4, 4])
    m.nets[1]["q_fc_0/w"] = torch.zeros(160, 32)
    with pytest.raises(ValueError):
        QLayout.from_iql(m, [0, 12, 32], 32)


@pytest.mark.parametrize("agent", ["iqll", "iqld"])
def test_monaco_tables_of_iql_agents_equal_the_net_file(agent, tmp_path):
    from deeprl_signal_control_b200.net import real_net as rn
    from deeprl_signal_control_b200.net.tables import NetTables
    net_file = str(tmp_path / "most.net.xml")
    with gzip.open(os.path.join(GOLD, "monaco_sumo", "most.net.xml.gz"), "rb") as fi, open(net_file, "wb") as fo:
        shutil.copyfileobj(fi, fo)
    a = rn.real_net_tables(agent)                 # no net file: the shipped cache
    b = rn.build_real_net(net_file, agent=agent)
    for k in NetTables._ARRAYS:
        x, y = np.asarray(getattr(a, k)), np.asarray(getattr(b, k))
        assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y), k
    for k in rn._LIST_FIELDS:
        assert [v for v in getattr(a, k)] == [v for v in getattr(b, k)], k
    assert a.neighbor_map == b.neighbor_map and a.phases == b.phases and a.max_na == b.max_na
    assert a.n_w_ls == [0] * 28 and a.n_f_ls == [0] * 28


def test_evaluate_script_maps_agent_names_like_main():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    try:
        import evaluate
    finally:
        sys.path.pop(0)
    assert evaluate.iql_model_type("iqld") == "dqn"
    assert evaluate.iql_model_type("iqll") == "lr"
    assert evaluate.iql_model_type("iql") == "lr"            # main.py: every other name is IQL-LR
