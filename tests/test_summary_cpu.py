"""CPU: the TensorBoard event log of the training driver (agents/summary.py, agents/train.py:Summaries) — CRC32C and the
TFRecord framing, a write / read round trip, the same file read by tensorboard's EventAccumulator, the tags and steps of
ia2c, ma2c, ia2c-fc, iqll and iqld against a step-by-step restatement of the reference's Trainer.run + backward,
scripts/extract_summaries.py, and rank 0's sum of the partial A2C records of two gloo ranks.

What the reference writes (quoted):
  agents/policies.py:62-72   if self.name.endswith('_0a'): summaries.append(tf.summary.scalar('loss/%s_policy_loss' %
                             self.name, policy_loss)) ... 'loss/%s_value_loss' ... 'loss/%s_total_loss' ...
                             'train/%s_gradnorm' % self.name, self.grad_norm
  agents/policies.py:331-338 'train/%s_loss' ... 'train/%s_q', tf.reduce_mean(q0) ... 'train/%s_tq', tf.reduce_mean(tq)
                             ... 'train/%s_gradnorm'
  agents/models.py:337-345   for k in range(10): ... summary_writer=summary_writer, global_step=global_step + k
  agents/models.py:333-335   if self.trans_buffer_ls[0].size < self.trans_buffer_ls[0].batch_size: return
  utils.py:288-291           global_step = self.global_counter.cur_step; self.model.backward(R, self.summary_writer,
                             global_step)
  utils.py:265-274, 306      self._add_summary(avg_reward, global_step, is_train=False) (avg of the per-seed means);
                             self._add_summary(mean_reward, global_step)
"""
import datetime
import os
import socket
import struct
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import torch

from deeprl_signal_control_b200.agents import summary as S
from deeprl_signal_control_b200.agents import train as drv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_crc32c_rfc3720_vector():
    assert S.crc32c(b"123456789") == 0xE3069283
    assert S.crc32c(b"") == 0
    assert S.crc32c(bytes(32)) == 0x8A9136AA                        # RFC 3720 B.4: 32 bytes of zeroes


def _write(tmp_path):
    w = S.SummaryWriter(str(tmp_path))
    w.add_scalar("train_reward", -412.5, 720, wall_time=1000.25)
    w.add_scalars({"loss/lstm_0a_policy_loss": 0.125, "train/lstm_0a_gradnorm": 3.0e-3}, 120, wall_time=1001.0)
    w.add_scalar("test_reward", float(np.float32(-1.1)), 0)
    w.add_scalar("train/dqn_0a_q", 1e30, 2 ** 40)
    w.close()
    return w.path


def test_round_trip(tmp_path):
    path = _write(tmp_path)
    name = os.path.basename(path)
    assert name.startswith("events.out.tfevents.") and name.endswith("." + socket.gethostname())
    recs = S.read_records(path)
    assert len(recs) == 5
    wt, step, version, values = S.decode_event(recs[0])
    assert version == "brain.Event:2" and values == []
    got = S.read_scalars(path)
    assert got["train_reward"] == [(1000.25, 720, -412.5)]
    assert got["loss/lstm_0a_policy_loss"] == [(1001.0, 120, 0.125)]
    assert got["train/lstm_0a_gradnorm"] == [(1001.0, 120, float(np.float32(3.0e-3)))]
    assert got["test_reward"][0][1:] == (0, float(np.float32(-1.1)))
    assert got["train/dqn_0a_q"][0][1:] == (2 ** 40, float(np.float32(1e30)))
    # a second writer in the same second does not overwrite the first file
    w2 = S.SummaryWriter(str(tmp_path))
    w2.close()
    assert w2.path != path and len(S.event_files(str(tmp_path))) == 2


def test_both_checksums_are_checked(tmp_path):
    path = _write(tmp_path)
    data = bytearray(open(path, "rb").read())
    n = struct.unpack("<Q", bytes(data[:8]))[0]
    for pos in (3, 12 + n // 2):                                    # in the length, in the first record's data
        bad = bytearray(data)
        bad[pos] ^= 0x01
        p = tmp_path / ("bad%d" % pos)
        p.write_bytes(bytes(bad))
        with pytest.raises(ValueError, match="checksum"):
            S.read_scalars(str(p))
    p = tmp_path / "cut"
    p.write_bytes(bytes(data[:-3]))
    with pytest.raises(ValueError, match="truncated"):
        S.read_scalars(str(p))


def test_tensorboard_reads_the_file(tmp_path):
    ea_mod = pytest.importorskip("tensorboard.backend.event_processing.event_accumulator")
    path = _write(tmp_path)
    ea = ea_mod.EventAccumulator(path, size_guidance={"scalars": 0})
    ea.Reload()
    mine = S.read_scalars(path)
    assert sorted(ea.Tags()["scalars"]) == sorted(mine)
    for tag, rows in mine.items():
        got = [(e.wall_time, e.step, e.value) for e in ea.Scalars(tag)]
        assert [(s, np.float32(v)) for _, s, v in got] == [(s, np.float32(v)) for _, s, v in rows], tag
        assert [w for w, _, _ in got] == [w for w, _, _ in rows]


# ---- the schedule of tags and steps ------------------------------------------------------------------------------
def reference_events(total_step, test_step, T, n_step, run_test, iql, buffer_size=None):
    """utils.py:Counter + Trainer.run + explore + the models' backward, one control step at a time: [(what, step)],
    what in {'update', 'round k', 'train_reward', 'test_reward'}.  IQL's batch_size is n_step (agents/models.py:
    ReplayBuffer(buffer_size, self.n_step)) and its buffer size is min(buffer_size, cum_size)."""
    cur = cur_test = cum = 0
    out = []
    while not cur >= total_step:
        if run_test and cur - cur_test >= test_step:
            cur_test = cur
            out.append(("test_reward", cur))
        t, done = 0, False
        while not done:
            for _ in range(n_step):
                cur += 1
                t += 1
                cum += 1
                done = t == T
                if done:
                    break
            global_step = cur
            if not iql:
                out.append(("update", global_step))
            elif min(buffer_size, cum) >= n_step:
                out += [("round %d" % k, global_step + k) for k in range(10)]
        out.append(("train_reward", cur))
    return out


class StubTrainer:
    """A batched trainer's interface to the driver, with a deterministic record per update: A2C [n_upd, 4], IQL
    [n_upd, 10, A, 4]; an IQL update runs once the ring holds batch_size (= n_step) entries."""

    def __init__(self, T, n_step, iql, R=3, A=2, buffer_size=None, partial=1.0):
        self.T_episode, self.n_step, self.iql, self.buffer_size = T, n_step, iql, buffer_size
        n_upd = -(-T // n_step)
        self.summary_rec = torch.zeros((n_upd, 10, A, 4) if iql else (n_upd, 4))
        self.summary_ran = np.zeros(n_upd, bool) if iql else np.ones(n_upd, bool)
        self.greward_trace = torch.zeros(T, R)
        self.episode_rewards, self.episode, self.cum, self.partial = [], 0, 0, partial

    def run(self, n):
        assert n == self.T_episode
        self.episode += 1
        for j in range(len(self.summary_ran)):
            self.cum += min(self.n_step, self.T_episode - j * self.n_step)
            v = 1000.0 * self.episode + j
            if self.iql:
                self.summary_ran[j] = min(self.buffer_size, self.cum) >= self.n_step
                if self.summary_ran[j]:
                    k = torch.arange(10, dtype=torch.float32)[:, None, None]
                    self.summary_rec[j] = v + 0.25 * k + torch.tensor([0.0, 0.5, 0.75, 0.125]) + \
                        100.0 * torch.arange(self.summary_rec.shape[2])[None, :, None]
            elif self.summary_rec is not None:
                self.summary_rec[j] = self.partial * torch.tensor([v, -0.5 * v, 0.25, 3.0 + j])
        self.greward_trace.copy_(-torch.arange(self.greward_trace.numel(), dtype=torch.float32).reshape(
            self.greward_trace.shape) * self.episode)
        self.episode_rewards.append(float(self.greward_trace.double().mean()))


class StubEvaluator:
    test_num = 2

    def __init__(self):
        self.calls = 0

    def perform_all(self):
        self.calls += 1
        return np.array([-1.0, -2.5]) * self.calls, np.array([0.5, 0.25])


TAGS = {
    "a2c": ["loss/{n}_policy_loss", "loss/{n}_value_loss", "loss/{n}_total_loss", "train/{n}_gradnorm"],
    "iql": ["train/{n}_loss", "train/{n}_q", "train/{n}_tq", "train/{n}_gradnorm"],
}
AGENTS = [("ia2c", "lstm", None, "lstm_0a"), ("ma2c", "lstm", None, "fplstm_0a"), ("ia2c", "fc", None, "fc_0a"),
          ("ma2c", "fc", None, "fpfc_0a"), ("iqll", "lstm", "lr", "lr_0a"), ("iqld", "lstm", "dqn", "dqn_0a")]


def _drive(tmp_path, agent, policy, model_type, total_step, test_step, T, n_step, run_test, buffer_size=1000):
    iql = agent.startswith("iq")
    name = S.summary_name(agent, policy, model_type)
    tr = StubTrainer(T, n_step, iql, buffer_size=buffer_size)
    w = S.SummaryWriter(str(tmp_path))
    summ = drv.Summaries(w, name, "iql" if iql else "a2c", n_step)
    d = drv.Trainer(tr, StubEvaluator(), drv.Counter(total_step, test_step, 10 ** 9), agent, run_test,
                    str(tmp_path) + "/", summary=summ)
    d.run()
    w.close()
    return name, d, [S.decode_event(r) for r in S.read_records(w.path)[1:]]


@pytest.mark.parametrize("agent,policy,model_type,name", AGENTS)
@pytest.mark.parametrize("total_step,test_step,T,n_step,run_test", [
    (360, 240, 120, 120, True),         # the GPU tests' shape: one A2C update per episode set
    (1000, 250, 120, 40, True),         # several updates per episode set, tests between them
    (300, 50, 120, 20, False),          # total_step not a multiple of T
    (240, 0, 120, 30, True),            # a test before every episode set, the first at step 0
])
def test_tags_and_steps_match_the_reference_run(tmp_path, agent, policy, model_type, name, total_step, test_step, T,
                                                n_step, run_test):
    iql = agent.startswith("iq")
    assert name == S.summary_name(agent, policy, model_type)
    got_name, d, events = _drive(tmp_path, agent, policy, model_type, total_step, test_step, T, n_step, run_test)
    want = reference_events(total_step, test_step, T, n_step, run_test, iql, buffer_size=1000)
    tags = [t.format(n=name) for t in TAGS["iql" if iql else "a2c"]]
    got, k_in_update = [], 0
    for wt, step, _, values in events:
        keys = [k for k, _ in values]
        if keys == ["train_reward"] or keys == ["test_reward"]:
            got.append((keys[0], step))
            k_in_update = 0
            continue
        assert keys == tags
        if iql:
            got.append(("round %d" % k_in_update, step))
            k_in_update = (k_in_update + 1) % 10
        else:
            got.append(("update", step))
    assert got == want
    # train_reward is the training row's avg_reward, test_reward the mean of the test's per-seed means
    rows = [r for r in d.data if r["test_id"] == -1]
    assert [v for _, _, _, vals in events for k, v in vals if k == "train_reward"] == \
        [float(np.float32(r["avg_reward"])) for r in rows]
    tests = pd.DataFrame([r for r in d.data if r["test_id"] >= 0])
    if len(tests):
        assert [v for _, _, _, vals in events for k, v in vals if k == "test_reward"] == \
            [float(np.float32(x)) for x in tests.groupby("step", sort=False).avg_reward.mean()]


@pytest.mark.parametrize("agent,model_type", [("iqll", "lr"), ("iqld", "dqn")])
def test_iql_writes_no_update_before_the_buffer_holds_a_batch(tmp_path, agent, model_type):
    # buffer_size < batch_size: the reference's size check (agents/models.py:333-335) skips every backward
    _, d, events = _drive(tmp_path, agent, "lstm", model_type, 360, 240, 120, 20, True, buffer_size=10)
    assert reference_events(360, 240, 120, 20, True, True, buffer_size=10) == \
        [("train_reward", 120), ("train_reward", 240), ("test_reward", 240), ("train_reward", 360)]
    assert [(vals[0][0], step) for _, step, _, vals in events] == \
        [("train_reward", 120), ("train_reward", 240), ("test_reward", 240), ("train_reward", 360)]


def test_record_values_go_to_their_tags(tmp_path):
    name, _, events = _drive(tmp_path, "ma2c", "lstm", None, 240, 10 ** 9, 120, 40, False)
    ev = [(step, dict(vals)) for _, step, _, vals in events if "train_reward" not in dict(vals)]
    for e, (step, vals) in enumerate(ev):
        ep, j = divmod(e, 3)
        v = 1000.0 * (ep + 1) + j
        p, vl, ent, g = np.float32(v), np.float32(-0.5 * v), np.float32(0.25), np.float32(3.0 + j)
        assert step == 120 * ep + 40 * (j + 1)
        assert vals == {"loss/%s_policy_loss" % name: p, "loss/%s_value_loss" % name: vl,
                        "loss/%s_total_loss" % name: np.float32(np.float32(p + vl) + ent),
                        "train/%s_gradnorm" % name: g}
    name, _, events = _drive(tmp_path / "q", "iqld", "lstm", "dqn", 120, 10 ** 9, 120, 60, False)
    ev = [(step, dict(vals)) for _, step, _, vals in events if "train_reward" not in dict(vals)]
    assert len(ev) == 20
    for e, (step, vals) in enumerate(ev):
        j, k = divmod(e, 10)
        base = 1000.0 + j + 0.25 * k                                # agent 0 only
        assert step == 60 * (j + 1) + k
        assert vals == {"train/dqn_0a_loss": np.float32(base), "train/dqn_0a_q": np.float32(base + 0.5),
                        "train/dqn_0a_tq": np.float32(base + 0.75), "train/dqn_0a_gradnorm": np.float32(base + 0.125)}


def test_summaries_off_changes_nothing(tmp_path):
    tr = StubTrainer(120, 40, False)
    tr.summary_rec = None
    d = drv.Trainer(tr, StubEvaluator(), drv.Counter(240, 120, 100), "ia2c", True, str(tmp_path) + "/")
    d.run()
    assert sorted(os.listdir(tmp_path)) == ["train_reward.csv"]


def test_extract_summaries_script(tmp_path):
    log = tmp_path / "log"
    w = S.SummaryWriter(str(log))
    for s in (120, 240, 360):
        w.add_scalar("train_reward", -float(s) / 3, s, wall_time=5000.0 + s)
        w.add_scalar("loss/fplstm_0a_value_loss", 0.5 / s, s, wall_time=5000.5 + s)
    w.close()
    for tag in ("train_reward", "loss/fplstm_0a_value_loss"):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "extract_summaries.py"), "--log-dir", str(log),
                            "--scalar-name", tag], capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stdout + r.stderr
        df = pd.read_csv(log / (tag + ".csv"), index_col=0, float_precision="round_trip")
        assert list(df.columns) == ["wall_time", "step", "value"]
        want = S.read_scalars(w.path)[tag]
        assert list(df.step) == [120, 240, 360]
        assert list(zip(df.wall_time, df.step, df.value)) == want
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "extract_summaries.py"), "--log-dir",
                        str(tmp_path / "model")], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode != 0


# ---- two gloo ranks ---------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    sys.path.insert(0, ROOT)
    from deeprl_signal_control_b200 import dist as D
    from deeprl_signal_control_b200.agents import summary as S_
    from deeprl_signal_control_b200.agents import train as drv_
    # the float64 rank-order sum on rank 0 only
    x = np.array([[1.0, 2.0], [3.0, 1e-8]], np.float32) * (rank + 1)
    got = D.sum_partials(x, group=None)
    if rank == 0:
        assert np.array_equal(got, x.astype(np.float64) * 3)
    else:
        assert got is None
    # the driver loop: each rank's A2C loss terms are its partial sum (here rank k holds (k + 1) / 3 of the whole);
    # the gradient norm is the same on every rank
    tr = StubTrainer(120, 40, False, partial=(rank + 1) / 3.0)
    orig_run = tr.run

    def run(n):
        orig_run(n)
        tr.summary_rec[:, 3] = 3.0 + torch.arange(3, dtype=torch.float32)     # global after the all-reduce
    tr.run = run
    w = S_.SummaryWriter(os.path.join(out_dir, "log")) if rank == 0 else None
    summ = drv_.Summaries(w, "fplstm_0a", "a2c", 40)
    d = drv_.Trainer(tr, StubEvaluator() if rank == 0 else None, drv_.Counter(240, 10 ** 9, 100), "ma2c", False,
                     os.path.join(out_dir, "data") + "/", group=dist.group.WORLD, summary=summ)
    if rank == 0:
        os.makedirs(os.path.join(out_dir, "data"), exist_ok=True)
    d.run()
    if w is not None:
        w.close()
    dist.destroy_process_group()


def test_rank0_sums_partial_a2c_records_of_two_gloo_ranks(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    files = S.event_files(str(tmp_path / "log"))
    assert len(files) == 1                                          # rank 1 writes no file
    got = S.read_scalars(files[0])
    for ep in (1, 2):
        for j in range(3):
            v = 1000.0 * ep + j
            step = 120 * (ep - 1) + 40 * (j + 1)
            p = [x for x in got["loss/fplstm_0a_policy_loss"] if x[1] == step]
            vl = [x for x in got["loss/fplstm_0a_value_loss"] if x[1] == step]
            g = [x for x in got["train/fplstm_0a_gradnorm"] if x[1] == step]
            # 1/3 + 2/3 of the whole: each part rounded to float32 on its rank, added in float64 on rank 0
            assert len(p) == 1 and p[0][2] == pytest.approx(v, rel=1e-6)
            assert vl[0][2] == pytest.approx(-0.5 * v, rel=1e-6)
            assert g[0][2] == float(np.float32(3.0 + j))
    assert [s for _, s, _ in got["train_reward"]] == [120, 240]


def test_iql_backward_honours_summary_writer(tmp_path):
    """IQL.backward(summary_writer, global_step) (the reference's one-environment protocol): agent 0's loss, mean q, mean
    tq and gradient norm of round k at global_step + k; nothing before the buffer holds a batch."""
    import configparser
    from deeprl_signal_control_b200.agents.models import IQL
    cp = configparser.ConfigParser()
    cp.read_string("""[MODEL_CONFIG]
max_grad_norm = 40
gamma = 0.99
lr_init = 1e-4
lr_decay = constant
epsilon_init = 1.0
epsilon_min = 0.01
epsilon_decay = constant
epsilon_ratio = 0.5
num_fc = 16
num_h = 8
batch_size = 4
buffer_size = 100
reward_norm = 10.0
reward_clip = 2.0
""")
    m = IQL([3, 5], [2, 3], [0, 2], 1000, cp["MODEL_CONFIG"], seed=1, model_type="dqn", device="cpu")
    rng = np.random.RandomState(0)
    w = S.SummaryWriter(str(tmp_path))
    m.backward(w, 3)                                                # empty buffer: skipped
    for _ in range(6):
        obs = [rng.rand(3), rng.rand(5)]
        m.add_transition(obs, [1, 2], [-3.0, -1.0], [rng.rand(3), rng.rand(5)], False)
    seen = []
    orig = m.td_update

    def td_update(i, *a):
        out = orig(i, *a)
        if i == 0:
            seen.append((out[0], float(m.td_means[0]), float(m.td_means[1]), out[1]))
        return out
    m.td_update = td_update
    m.backward(w, 6)
    w.close()
    got = S.read_scalars(w.path)
    assert sorted(got) == ["train/dqn_0a_gradnorm", "train/dqn_0a_loss", "train/dqn_0a_q", "train/dqn_0a_tq"]
    for j, tag in enumerate(("loss", "q", "tq", "gradnorm")):
        rows = got["train/dqn_0a_%s" % tag]
        assert [s for _, s, _ in rows] == list(range(6, 16))
        assert [v for _, _, v in rows] == [float(np.float32(x[j])) for x in seen]
