"""Scenario envs with the reference's names, and the two constructors the entry points share (scripts/train.py,
scripts/evaluate.py): `make_env` picks the env class from `[ENV_CONFIG]` as main.py:init_env does, `greedy_controller`
the scenario's greedy policy."""


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
