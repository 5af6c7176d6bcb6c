"""Scenario envs with the reference's names, and the two constructors the entry points share (scripts/train.py,
scripts/evaluate.py): `make_env` picks the env class from `[ENV_CONFIG]` as main.py:init_env does, `greedy_controller`
the scenario's greedy policy, `maxpressure_controller` the max-pressure one, `fixedtime_controller` the fixed-time
one, `actuated_controller` the vehicle-actuated one."""


# the [ENV_CONFIG] keys that set each scenario's traffic demand and nothing else: two configs that differ only in these
# build nets that differ only in net.tables.DEMAND_FIELDS, which one simulator takes per replica
# (BatchedSim.set_replica_demand).  SUMO-file scenarios (any other scenario name with a `net_file`) take `route_file`,
# accepted only where the other route file keeps every route and source (`check_demand_tables`).
DEMAND_KEYS = {
    'large_grid': ('peak_flow1', 'peak_flow2'),
    'real_net': ('flow_rate',),
    'small_grid': ('num_extra_car_per_hour',),
}
SUMO_FILE_DEMAND_KEYS = ('route_file',)


def demand_keys(cfg):
    """The demand keys (DEMAND_KEYS) of an `[ENV_CONFIG]` section's scenario; () for an unknown scenario."""
    scen = cfg.get('scenario')
    if scen in DEMAND_KEYS:
        return DEMAND_KEYS[scen]
    return SUMO_FILE_DEMAND_KEYS if cfg.get('net_file', fallback=None) else ()


def parse_demand(text, option='--demand'):
    """'k=v,k=v' -> {k: v} (in the given order), the value of the command-line `option` that names one demand level.
    Refuses an empty level, a pair without '=' and a repeated key."""
    out = {}
    for pair in text.split(","):
        pair = pair.strip()
        if not pair:
            continue
        key, sep, val = pair.partition("=")
        key, val = key.strip(), val.strip()
        if not sep or not key or not val:
            raise ValueError("%s takes KEY=VALUE pairs separated by ',' (got %r)" % (option, text))
        if key in out:
            raise ValueError("%s %r names %s twice" % (option, text, key))
        out[key] = val
    if not out:
        raise ValueError("%s %r names no key" % (option, text))
    return out


def demand_label(level):
    """The directory name of a demand level: its key-value pairs joined by '_' (peak_flow1-1400_peak_flow2-1180)."""
    import os
    return "_".join("%s-%s" % (k, os.path.basename(v) if k == "route_file" else v) for k, v in level.items())


def check_demand_tables(base, other, what, ignore=()):
    """Refuse (ValueError naming `what` and the field) two nets that differ in more than their demand tables."""
    from ..net.tables import DEMAND_FIELDS, demand_mismatch
    f = demand_mismatch(base, other, ignore=ignore)
    if f is not None:
        raise ValueError('%s: the net differs in %r, not only in its demand (%s)' % (what, f, ', '.join(DEMAND_FIELDS)))


def make_env(cfg, n_replicas, output_path, is_record=True, device=0):
    """The scenario env of an `[ENV_CONFIG]` section (large_grid, real_net, small_grid, or a SUMO-file scenario through
    `net_file`) with `n_replicas` lock-stepped replicas."""
    scen = cfg.get("scenario")
    if scen == "large_grid":
        from .large_grid_env import LargeGridEnv as Env
    elif scen == "real_net":
        from .real_net_env import RealNetEnv as Env
    elif scen == "small_grid":
        from .small_grid_env import SmallGridEnv as Env
    elif cfg.get("net_file", fallback=None):
        from .sumo_env import SumoNetEnv as Env
    else:
        raise ValueError("unknown scenario %r" % scen)
    return Env(cfg, output_path=output_path, is_record=is_record, record_stat=False, n_replicas=n_replicas,
               device=device)


def greedy_controller(env):
    from .large_grid_env import LargeGridController
    from .real_net_env import RealNetController
    from .small_grid_env import SmallGridController
    from .sumo_env import SumoNetController
    if env.name == "large_grid":
        return LargeGridController(env.node_names)
    if env.name == "real_net":
        return RealNetController(env.node_names, env.nodes)
    if env.name == "small_grid":
        return SmallGridController(env.node_names)
    return SumoNetController(env.node_names, env.nodes, {n: env.phase_map.phases[n].phases for n in env.node_names})


def maxpressure_controller(env):
    """The max-pressure controller (envs.maxpressure) of any scenario env: `name = 'maxpressure'`."""
    from .maxpressure import MaxPressureController
    return MaxPressureController(env)


def fixedtime_controller(env):
    """The fixed-time controller (envs.fixedtime) of any scenario env, `name = 'fixedtime'`; puts the env's simulator
    into fixed mode, every replica running the env's signal programs."""
    from .fixedtime import FixedTimeController
    ctrl = FixedTimeController(env)
    env._ensure_sim().set_signal_program(ctrl.program)
    return ctrl


def actuated_controller(env):
    """The vehicle-actuated controller (envs.actuated) of any scenario env, `name = 'actuated'`; puts the env's
    simulator into actuated mode, every replica running the env's actuated programs."""
    from .actuated import ActuatedController
    ctrl = ActuatedController(env)
    env._ensure_sim().set_actuated_program(ctrl.program)
    return ctrl
