"""GPU parity: CUDA control-step kernel (through the C ABI) vs the CPU oracle, bit-exact.

Integer outputs (vehicle counts, halting counts, head waits, phases, done) and the full
per-vehicle state must be identical; float outputs (obs, rewards) are produced by the same
IEEE-binary32 operation sequence on both sides, so they are compared bit-for-bit too.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(net, par, R):
    from deeprl_signal_control_b200.sim import BatchedSim
    from oracle.sim_ref import RefSim
    return BatchedSim(net, par, R), RefSim(net, par, R)


def _compare_step(gpu, ref, act, fp, check_state_of=()):
    a_dev = torch.from_numpy(act).cuda()
    fp_dev = None if fp is None else torch.from_numpy(fp).cuda()
    obs, rew, grew, done = gpu.step(a_dev, fp_dev)
    o2, r2, g2, d2 = ref.step(act, fp)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(obs.cpu().numpy().view(np.uint32), o2.view(np.uint32))
    np.testing.assert_array_equal(rew.cpu().numpy().view(np.uint32), r2.view(np.uint32))
    np.testing.assert_array_equal(grew.cpu().numpy().view(np.uint32), g2.view(np.uint32))
    np.testing.assert_array_equal(done.cpu().numpy(), d2)
    for a, b in zip(gpu.counts(), ref.counts()):
        np.testing.assert_array_equal(a.cpu().numpy(), b)
    for r in check_state_of:
        c1, v1 = gpu.dump_state(r)
        c2, v2 = ref.dump_state(r)
        np.testing.assert_array_equal(c1, c2)
        np.testing.assert_array_equal(v1, v2)


@pytest.mark.parametrize("agent", ["ma2c", "ia2c", "greedy"])
def test_random_actions_bit_exact(agent):
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import EnvParams
    net, par = build_large_grid(agent=agent), EnvParams(agent=agent)
    R = 6
    gpu, ref = _mk(net, par, R)
    seeds = np.arange(100, 100 + R, dtype=np.uint64) * np.uint64(7919)
    gpu.reset(seeds); ref.reset(seeds)
    np.testing.assert_array_equal(gpu.observe().cpu().numpy(), ref.observe())
    rng = np.random.default_rng(1)
    for step in range(260):
        act = rng.integers(0, 5, size=(R, net.n_nodes), dtype=np.int32)
        fp = None
        if agent == "ma2c":
            fp = rng.random((R, net.n_nodes, net.max_na), dtype=np.float32)
        _compare_step(gpu, ref, act, fp, check_state_of=(0, R - 1) if step % 20 == 0 else ())
    assert ref.misc(0)["live"] > 50  # the comparison covered a loaded network


def test_full_episode_greedy_bit_exact(grid_ma2c):
    """720 control steps (one whole 3600-s episode, peak demand, arrivals, done flag)."""
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import EnvParams
    net, par = build_large_grid(agent="greedy"), EnvParams(agent="greedy")
    R = 3
    gpu, ref = _mk(net, par, R)
    seeds = np.array([12, 13, 10000], dtype=np.uint64)
    gpu.reset(seeds); ref.reset(seeds)
    gpu.set_train_mode(False); ref.set_train_mode(False)
    ob = ref.observe()
    dones = []
    for step in range(720):
        o = ob.reshape(R, net.n_nodes, 6)
        flows = np.stack([o[..., 0] + o[..., 3], o[..., 2] + o[..., 5], o[..., 1] + o[..., 4],
                          o[..., 1] + o[..., 2], o[..., 4] + o[..., 5]], -1)
        act = flows.argmax(-1).astype(np.int32)          # envs/large_grid_env.py:56-60
        _compare_step(gpu, ref, act, None, check_state_of=(1,) if step % 60 == 0 else ())
        ob = gpu.obs.cpu().numpy()
        dones.append(int(gpu.done[0]))
    assert dones[-1] == 1 and sum(dones) == 1
    m = ref.misc(0)
    assert m["departed"] > 3500 and m["arrived"] > 3000


def test_host_entry_point_matches_device_entry_point(grid_ma2c):
    net, par = grid_ma2c
    from deeprl_signal_control_b200.sim import BatchedSim
    R = 4
    a, b = BatchedSim(net, par, R), BatchedSim(net, par, R)
    seeds = np.arange(R, dtype=np.uint64) + np.uint64(5)
    a.reset(seeds); b.reset(seeds)
    rng = np.random.default_rng(3)
    for _ in range(40):
        act = rng.integers(0, 5, size=(R, net.n_nodes), dtype=np.int32)
        fp = rng.random((R, net.n_nodes, net.max_na), dtype=np.float32)
        o1, r1, g1, d1 = a.step(torch.from_numpy(act).cuda(), torch.from_numpy(fp).cuda())
        o2, r2, g2, d2 = b.step_host(act, fp)
        np.testing.assert_array_equal(o1.cpu().numpy(), o2)
        np.testing.assert_array_equal(r1.cpu().numpy(), r2)
        np.testing.assert_array_equal(g1.cpu().numpy(), g2)


def test_traffic_stats_match_state_dump(grid_ma2c):
    """tsc_get_traffic_stats (envs/env.py:409-437) against the same quantities computed from the state dump."""
    net, par = grid_ma2c
    from deeprl_signal_control_b200.sim import BatchedSim
    R = 3
    sim = BatchedSim(net, par, R)
    sim.reset(np.arange(R, dtype=np.uint64) + np.uint64(77))
    rng = np.random.default_rng(9)
    for _ in range(150):
        sim.step(torch.from_numpy(rng.integers(0, 5, (R, net.n_nodes), dtype=np.int32)).cuda())
    st = sim.traffic_stats().cpu().numpy()
    for r in range(R):
        cnt, veh = sim.dump_state(r)
        spd = veh[:, 1].copy().view(np.float32); wait = (veh[:, 2] & 1023).astype(np.float64)
        lane_of = np.repeat(np.arange(net.n_lanes), cnt)
        halt = np.bincount(lane_of[spd < 0.1], minlength=net.n_lanes)[net.det_lane]
        assert st[r, 0] == len(veh) and len(veh) > 50
        np.testing.assert_allclose(st[r, 3], wait.mean(), rtol=1e-5)
        np.testing.assert_allclose(st[r, 4], spd.mean(), rtol=1e-4)
        np.testing.assert_allclose(st[r, 5], halt.mean(), rtol=1e-5)
        np.testing.assert_allclose(st[r, 6], halt.std(), rtol=1e-3, atol=1e-4)
        assert st[r, 1] - st[r, 2] == len(veh)          # departed - arrived = live


def test_gridlock_full_rings_and_teleport_bit_exact():
    """Edge cases of the junction logic: one phase held for minutes (red approaches fill their lanes to capacity,
    transfers are refused, source backlogs grow), a short teleport threshold so that heads waiting longer than
    `teleport_sec` ignore the signal (envs/env.py:281-284, SURVEY App. A), then random actions to drain."""
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import EnvParams
    net, par = build_large_grid(agent="ia2c"), EnvParams(agent="ia2c", teleport_sec=45)
    R = 4
    gpu, ref = _mk(net, par, R)
    seeds = np.array([1, 2, 3, 4], dtype=np.uint64)
    gpu.reset(seeds); ref.reset(seeds)
    rng = np.random.default_rng(9)
    full_seen = teleport_seen = False
    for step in range(420):
        if step < 300:
            act = np.full((R, net.n_nodes), 3 if step < 150 else 4, np.int32)      # one approach green only
        else:
            act = rng.integers(0, 5, size=(R, net.n_nodes), dtype=np.int32)
        _compare_step(gpu, ref, act, None, check_state_of=(0, R - 1) if step % 30 == 0 else ())
        if step % 10 == 0:
            cnt, _ = ref.dump_state(0)
            full_seen |= bool((cnt >= net.lane_cap - 1).any())
            teleport_seen |= bool((ref.counts()[2] >= 45).any())
    assert full_seen and teleport_seen
    assert ref.misc(0)["backlog"] > 0


def test_single_replica_and_observe_only():
    """R = 1 (the reference's own configuration) and observe() without stepping leave the state untouched."""
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import EnvParams
    net, par = build_large_grid(agent="ma2c"), EnvParams(agent="ma2c")
    gpu, ref = _mk(net, par, 1)
    seeds = np.array([77], dtype=np.uint64)
    gpu.reset(seeds); ref.reset(seeds)
    rng = np.random.default_rng(3)
    for step in range(60):
        act = rng.integers(0, 5, size=(1, net.n_nodes), dtype=np.int32)
        fp = rng.random((1, net.n_nodes, net.max_na), dtype=np.float32)
        _compare_step(gpu, ref, act, fp, check_state_of=(0,) if step % 20 == 0 else ())
        if step % 15 == 0:
            c0, v0 = gpu.dump_state(0)
            o1 = gpu.observe(torch.from_numpy(fp).cuda()).cpu().numpy()
            np.testing.assert_array_equal(o1.view(np.uint32), ref.observe(fp).view(np.uint32))
            c1, v1 = gpu.dump_state(0)
            np.testing.assert_array_equal(c0, c1); np.testing.assert_array_equal(v0, v1)


def test_many_waves_and_replica_ranges_bit_exact():
    """R = 2304 replicas = several waves of resident CTAs (a few per SM x 132 SMs on an H100): the oracle follows a SAMPLE of
    replicas spread over all waves (each replica is independent, so stepping the sample alone is the same computation),
    and the host-buffer range entry point (`tsc_step_host_range`, rep0 > 0) must agree with the device-resident step."""
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import EnvParams
    from deeprl_signal_control_b200.sim import BatchedSim
    from oracle.sim_ref import RefSim
    net, par = build_large_grid(agent="ma2c"), EnvParams(agent="ma2c")
    R = 2304
    sample = np.array([0, 1, 591, 592, 593, 1183, 1184, 1500, 1776, 2047, 2048, 2302, 2303])
    gpu, gpu2 = BatchedSim(net, par, R), BatchedSim(net, par, R)
    ref = RefSim(net, par, len(sample))
    seeds = np.arange(R, dtype=np.uint64) * np.uint64(31) + np.uint64(5)
    gpu.reset(seeds); gpu2.reset(seeds); ref.reset(seeds[sample])
    rng = np.random.default_rng(3)
    r0, cnt = 1000, 700                                      # the range stepped through the host-buffer call
    for step in range(150):
        act = rng.integers(0, 5, size=(R, net.n_nodes), dtype=np.int32)
        fp = rng.random((R, net.n_nodes, net.max_na), dtype=np.float32)
        obs, rew, grew, done = gpu.step(torch.from_numpy(act).cuda(), torch.from_numpy(fp).cuda())
        o2, r2, g2, d2 = ref.step(act[sample], fp[sample], threads=4)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(obs[sample].cpu().numpy().view(np.uint32), o2.view(np.uint32))
        np.testing.assert_array_equal(rew[sample].cpu().numpy().view(np.uint32), r2.view(np.uint32))
        np.testing.assert_array_equal(grew[sample].cpu().numpy().view(np.uint32), g2.view(np.uint32))
        # second handle: replicas [r0, r0+cnt) through tsc_step_host_range, the rest through the device call on ranges
        ho = np.zeros((cnt, net.n_obs), np.float32); hr = np.zeros((cnt, net.n_nodes), np.float32)
        hg = np.zeros(cnt, np.float32); hd = np.zeros(cnt, np.uint8)
        gpu2.step_host_range(r0, cnt, np.ascontiguousarray(act[r0:r0 + cnt]), np.ascontiguousarray(fp[r0:r0 + cnt]),
                             ho, hr, hg, hd, sync=True)
        np.testing.assert_array_equal(ho.view(np.uint32), obs[r0:r0 + cnt].cpu().numpy().view(np.uint32))
        np.testing.assert_array_equal(hr.view(np.uint32), rew[r0:r0 + cnt].cpu().numpy().view(np.uint32))
        np.testing.assert_array_equal(hg.view(np.uint32), grew[r0:r0 + cnt].cpu().numpy().view(np.uint32))
    for k, r in enumerate(sample[[0, 3, 7, 12]]):
        c1, v1 = gpu.dump_state(int(r))
        c2, v2 = ref.dump_state([0, 3, 7, 12][k])
        np.testing.assert_array_equal(c1, c2)
        np.testing.assert_array_equal(v1, v2)
    c1, v1 = gpu.dump_state(r0 + 5)
    c2, v2 = gpu2.dump_state(r0 + 5)
    np.testing.assert_array_equal(c1, c2); np.testing.assert_array_equal(v1, v2)
    assert ref.misc(0)["live"] > 100


def test_initial_fleet_bit_exact():
    """init_density > 0 (large_grid/data/build_file.py:223-266): 120 extra demand sources on internal lanes, several
    sources per lane, 132 routes — CUDA vs oracle for the first 10 minutes (the fleet drains through the junctions)."""
    from deeprl_signal_control_b200.net.large_grid import build_large_grid
    from deeprl_signal_control_b200.net.tables import EnvParams
    net, par = build_large_grid(agent="ma2c", init_density=0.4, seed=12), EnvParams(agent="ma2c")
    R = 3
    gpu, ref = _mk(net, par, R)
    seeds = np.array([12, 13, 99], dtype=np.uint64)
    gpu.reset(seeds); ref.reset(seeds)
    rng = np.random.default_rng(5)
    for step in range(120):
        act = rng.integers(0, 5, size=(R, net.n_nodes), dtype=np.int32)
        fp = rng.random((R, net.n_nodes, net.max_na), dtype=np.float32)
        _compare_step(gpu, ref, act, fp, check_state_of=(0, 2) if step % 30 == 0 else ())
    m = ref.misc(0)
    assert m["departed"] > 120 * 12 * 0.9 and m["arrived"] > 200
