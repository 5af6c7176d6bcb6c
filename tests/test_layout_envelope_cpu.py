"""CPU: which forward and update path `BatchedA2C` takes for each layout (agents/learner.py:learner_paths), for the shipped
scenarios at the reference's model widths and for synthetic layouts at the edges of the kernels' input tile, and that
each choice meets the preconditions of the kernels it launches (tests/layout_envelope.py lists the layouts)."""
import os
import re

import pytest

from tests.layout_envelope import BEYOND, EDGES, ROOT, SCENARIOS, net_tables, scenario_layout, synthetic_layout


def _check_preconditions(lay, p):
    from deeprl_signal_control_b200.agents.learner import V2_DX
    mw = int(lay.n_wave.max())
    if p.forward == "v2":          # tscl_policy_step_v2 / _v2g / _pi: an instantiated dx and a 64-slot input tile
        assert lay.dx in V2_DX and lay.kw > 0
    if p.forward == "v1":          # tscl_policy_step stages a 32-wide wave block
        assert lay.kw == 32 and lay.dx % 16 == 0 and lay.dx <= 224
    if p.forward != "fp32":
        assert mw <= lay.kw
    if p.update == "lean":         # the tensor-core fc weight gradients carry the bias in the spare slot kw - 1
        assert p.fc_bwd_tc and mw < lay.kw and p.wgrad_tc and p.forward == "v2"
    if p.update == "store":        # the wave block fills its tile: SIMT fc weight gradients
        assert not p.fc_bwd_tc and mw == lay.kw and p.forward == "v2"
    if p.dx_fc_fused:              # tscl_dx_fc_bwd_tc: the v2 widths only
        assert lay.dx in V2_DX
    if p.update == "recompute":
        assert p.forward == "v1" and p.bwd_tc and p.wgrad_tc


def _check_population(lay, p):
    """K = 2 is accepted exactly where its forward (the grouped v2 launch) and its update (the store paths, each member
    with its own weights) exist"""
    from deeprl_signal_control_b200.agents.learner import learner_paths
    if p.tc_v2 and p.dx_fc_fused:
        q = learner_paths(lay, True, 2)
        assert q.update in ("lean", "store") and vars(q) == vars(p)
    else:
        with pytest.raises(ValueError, match="population"):
            learner_paths(lay, True, 2)


@pytest.mark.parametrize("scenario,agent,fw", list(SCENARIOS))
def test_scenario_paths(tmp_path, scenario, agent, fw):
    from deeprl_signal_control_b200.agents.learner import learner_paths
    lay = scenario_layout(net_tables(scenario, agent, str(tmp_path)), agent, fw)
    p = learner_paths(lay)
    assert (p.forward, p.update) == SCENARIOS[(scenario, agent, fw)], (lay.dx, lay.kw, vars(p))
    _check_preconditions(lay, p)
    _check_population(lay, p)
    off = learner_paths(lay, use_tc=False)
    assert (off.forward, off.update) == ("fp32", "fp32") and not any(
        getattr(off, k) for k in ("use_tc", "tc_v2", "dx_own", "dx_fc_fused", "bwd_tc", "fc_bwd_tc", "wgrad_tc"))


def test_monaco_ia2c_at_the_reference_widths():
    """config_ia2c_real.ini: no Monaco agent has wait inputs, so ft = 0 and dx = num_fw = 128; the widest wave block is
    34, so the tile is 48 | 16 and the v1 kernel cannot serve it: the v2 kernel is instantiated at dx = 128"""
    from deeprl_signal_control_b200.agents.learner import learner_paths
    lay = scenario_layout(net_tables("real_net", "ia2c"), "ia2c")
    assert (lay.ft, lay.dx, lay.kw, int(lay.n_wave.max())) == (0, 128, 48, 34)
    p = learner_paths(lay)
    assert p.forward == "v2" and p.update == "lean" and p.dx_fc_fused


@pytest.mark.parametrize("fw", [64, 96])
def test_v1_with_a_48_wide_wave_block_is_refused(fw):
    """Monaco IA2C at fc widths outside the v2 set would select the v1 forward, which stages 32 wave inputs: refused at
    construction with the supported widths named, rather than at the first forward"""
    from deeprl_signal_control_b200.agents.learner import learner_paths
    lay = scenario_layout(net_tables("real_net", "ia2c"), "ia2c", fw)
    assert lay.kw == 48 and lay.dx == fw
    with pytest.raises(ValueError, match=r"\(128, 160, 192, 224\)"):
        learner_paths(lay)
    assert learner_paths(lay, use_tc=False).forward == "fp32"


@pytest.mark.parametrize("name", list(EDGES))
def test_edge_paths(name):
    from deeprl_signal_control_b200.agents.learner import learner_paths
    kw, forward, update = EDGES[name]
    lay = synthetic_layout(**kw)
    p = learner_paths(lay)
    assert (p.forward, p.update) == (forward, update), (lay.dx, lay.kw, vars(p))
    _check_preconditions(lay, p)
    _check_population(lay, p)


def test_beyond_the_limits():
    """dx 240 with use_tc is refused by learner_paths; the other layouts one past a kernel limit leave the tensor-core
    paths (no 64-slot tile fits them) and are refused by tscl_create on the device (test_layout_envelope_gpu.py)"""
    from deeprl_signal_control_b200.agents.learner import learner_paths
    for name, (kw, msg) in BEYOND.items():
        lay = synthetic_layout(**kw)
        if name == "dx240":
            assert lay.dx == 240
            with pytest.raises(ValueError, match=msg):
                learner_paths(lay)
        elif name == "max_na9":
            assert lay.max_na == 9 and learner_paths(lay).forward == "v2"
        else:
            assert learner_paths(lay).forward in ("fp32", "v2")


def test_population_without_the_fused_dx_is_refused():
    from deeprl_signal_control_b200.agents.learner import learner_paths
    lay = scenario_layout(net_tables("large_grid", "ma2c"), "ma2c")
    assert not learner_paths(lay, dx_library=True).dx_fc_fused
    with pytest.raises(ValueError, match="TSC_DX_LIBRARY"):
        learner_paths(lay, True, 2, dx_library=True)


def test_v2_widths_match_the_kernel_instantiations():
    """learner.V2_DX is the dx set of P2_DX_OK, and every width in it has its forward (train, pi-only, grouped) and
    fused dX / fc weight-gradient instantiation"""
    from deeprl_signal_control_b200.agents.learner import V2_DX
    src = open(os.path.join(ROOT, "deeprl_signal_control_b200", "csrc", "tsc_policy_tc.cu")).read()
    ok = re.search(r"#define P2_DX_OK\(dx\) (.*)", src).group(1)
    assert tuple(sorted(int(x) for x in re.findall(r"\(dx\) == (\d+)", ok))) == V2_DX
    for dx in V2_DX:
        assert "P2_CASE(%d)" % dx in src
        assert "policy_step_tc2_kernel<%d, false, true>" % dx in src
        assert "policy_step_tc2_kernel<%d, false, false, true>" % dx in src
        assert "dx_fc_bwd_tc_kernel<%d>, cudaFuncAttributeMaxDynamicSharedMemorySize" % dx in src
