"""Tuning of fixed-time signal plans on the device: a cross-entropy search over the green durations and offsets of a
scenario's own static programs (envs.fixedtime), every candidate plan of a generation one member of one `_Group`.

    tune_fixedtime(config_path, base_dir, seeds, candidates=512, generations=30, elite_frac=0.1, min_green=5,
                   max_green=60, rng_seed=0, device=0)

Search space (`search_space`), from the env's own programs (envs.fixedtime.env_program, its `tll_file` applied):
- a green phase is one with at least one 'G' / 'g' link and no 'y' link; its duration is an integer in
  [min(min_green, d0), max(max_green, d0)], d0 the shipped duration, which is therefore always inside the bounds;
- every other phase (yellow, all-red) keeps its duration, and phase order and states are not changed;
- node i's offset is a fraction u in [0, 1) of the node's own cycle C_i (that of the candidate's durations):
  offset = floor(u * C_i).

Objective: the mean over the tuning seeds of each test-mode episode's mean step reward, `mean_reward` of
agents.evaluator.episode_summary, which scripts/evaluate.py reports for a `fixedtime` directory on those seeds.  The K
candidates of a generation run as K fixed-time members of one `_Group` (member p on replicas p * S .. (p + 1) * S - 1
through tsc_set_replica_signal_programs) on the env of the config with `test_seeds` set to the tuning seeds and
`is_record=False`, and their scores are those of `_Group.rewards()`.  The group is built once per run and the
members' programs are swapped between generations.

Cross-entropy method (`cem`), a diagonal Gaussian:
- the green means start at d0 and their stds at (hi - lo) / 4; the offset-fraction means at (offset0 mod C0) / C0 and
  their stds at 0.25;
- each generation draws, from numpy.random.Generator(PCG64(rng_seed)), a standard normal [K - 1, n_green] and then a
  standard normal [K - 1, n_nodes]; candidate k >= 1 takes greens clip(rint(mean + std * z), lo, hi) and offset
  fractions (mean + std * z) mod 1;
- candidate 0 is the incumbent, the best plan evaluated so far (in generation 0 the shipped plan, its offsets as
  shipped).  The objective is deterministic on fixed seeds, so from generation 1 on the incumbent's score must repeat
  bit for bit, and the search raises if it does not;
- the elites are the top max(1, round(elite_frac * K)) candidates (Python's round), ties going to the lower index; the
  new incumbent is the first candidate of the highest score, so it never gets worse;
- the green means and stds become the elites' arithmetic mean and (population) std; the offset fractions take the
  elites' circular mean and circular std sqrt(-2 ln Rbar) / (2 pi), Rbar the mean resultant length of the angles
  2 pi u; the stds are floored at 0.5 s for greens and 0.01 for offset fractions.

The run writes an agent directory `<base_dir>/fixedtime/` that the evaluation scripts run unchanged:
- data/<config name>: the config with [ENV_CONFIG] tll_file set to the absolute path of data/tuned.tll.xml (the
  config's other paths as given);
- data/tuned.tll.xml: every node's best program (envs.fixedtime.write_tll);
- data/tune_log.csv: one row per generation: generation, the incumbent's reward after it, the generation's best, mean
  and elite-mean reward, and the mean green and offset-fraction std the generation sampled with;
- data/tune.json: the settings, the seeds, the bounds, the shipped plan's score and the final score.
No wall-clock time goes into these files, so two runs write the same bytes; it goes to the log.  With generations = 0
the shipped plan is evaluated once (every member running it) and written as it is.
"""
from __future__ import annotations

import configparser
import csv
import json
import logging
import os
import time
from dataclasses import dataclass

import numpy as np

# the evaluation scripts' default seeds (scripts/evaluate_agents.py, the reference's main.py): never tuned on
EVALUATION_SEEDS = tuple(range(10000, 100001, 10000))
GREEN_STD_FLOOR, OFFSET_STD_FLOOR = 0.5, 0.01


@dataclass
class SearchSpace:
    """The searched part of a SignalProgram `base` (env node order): green phase j is phase `phase[j]` of node
    `node[j]`, its duration an integer in [lo[j], hi[j]], shipped d0[j]; every node's offset is searched."""
    base: object
    node: np.ndarray
    phase: np.ndarray
    lo: np.ndarray
    hi: np.ndarray
    d0: np.ndarray

    @property
    def n_green(self) -> int:
        return len(self.node)

    @property
    def n_nodes(self) -> int:
        return len(self.base.n_phases)

    def program(self, greens, offsets):
        """The SignalProgram of integer green durations [n_green] and integer offsets [n_nodes]."""
        from ..envs.fixedtime import SignalProgram
        b = self.base
        dur = b.dur.copy()
        dur[self.node, self.phase] = np.asarray(greens, np.int32)
        return SignalProgram(n_phases=b.n_phases.copy(), dur=dur, open=b.open.copy(), major=b.major.copy(),
                             yellow=b.yellow.copy(), offset=np.asarray(offsets, np.int32).copy())

    def cycles(self, greens) -> np.ndarray:
        """int64 [n_nodes]: each node's cycle under the green durations `greens`."""
        c = self.base.dur.sum(axis=1).astype(np.int64)
        np.add.at(c, self.node, np.asarray(greens, np.int64) - self.d0)
        return c


def search_space(program, min_green=5, max_green=60) -> SearchSpace:
    """The SearchSpace of a SignalProgram: its green phases (an open link and no yellow link) with their bounds."""
    node, phase = [], []
    for i, n_p in enumerate(program.n_phases):
        for k in range(int(n_p)):
            if program.open[i, k] and not program.yellow[i, k]:
                node.append(i); phase.append(k)
    node, phase = np.asarray(node, np.int64), np.asarray(phase, np.int64)
    d0 = program.dur[node, phase].astype(np.int64)
    return SearchSpace(base=program, node=node, phase=phase, lo=np.minimum(min_green, d0), hi=np.maximum(max_green, d0),
                       d0=d0)


def offsets_of(space, greens, fracs) -> np.ndarray:
    """int64 [n_nodes]: floor(u * C_i) of the offset fractions `fracs` on the cycles of `greens`."""
    c = space.cycles(greens)
    return np.minimum(np.floor(np.asarray(fracs, np.float64) * c).astype(np.int64), c - 1)


def circular_mean_std(u):
    """Circular mean in [0, 1) and circular std sqrt(-2 ln Rbar) / (2 pi) of fractions u [n, d] along axis 0."""
    a = 2.0 * np.pi * np.asarray(u, np.float64)
    s, c = np.sin(a).mean(axis=0), np.cos(a).mean(axis=0)
    mean = np.mod(np.arctan2(s, c) / (2.0 * np.pi), 1.0)
    rbar = np.sqrt(s * s + c * c)
    std = np.sqrt(-2.0 * np.log(np.maximum(rbar, 1e-300))) / (2.0 * np.pi)
    return mean, std


def n_elites(candidates, elite_frac) -> int:
    return max(1, int(round(elite_frac * candidates)))


def cem(space, objective, candidates=512, generations=30, elite_frac=0.1, rng_seed=0, on_generation=None):
    """The cross-entropy search of the module docstring.  `objective(greens [K][n_green] int64, offsets [K][n_nodes]
    int64)` returns float64 [K] scores.  Returns {'greens', 'offsets', 'scores': per generation [K] arrays, 'best_greens',
    'best_offsets', 'best_score', 'shipped_score', 'rows': one log row per generation}.  `on_generation(row)` is called
    after each generation."""
    K, G, N = int(candidates), space.n_green, space.n_nodes
    rng = np.random.Generator(np.random.PCG64(rng_seed))
    mg = space.d0.astype(np.float64)
    sg = (space.hi - space.lo).astype(np.float64) / 4.0
    c0 = space.cycles(space.d0)
    inc_g, inc_o = space.d0.copy(), np.asarray(space.base.offset, np.int64).copy()
    mu = np.mod(inc_o, c0) / c0
    su = np.full(N, 0.25)
    inc_u, inc_score = mu.copy(), None
    out = dict(greens=[], offsets=[], scores=[], rows=[], shipped_score=None)
    for gen in range(int(generations)):
        zg = rng.standard_normal((K - 1, G))
        zu = rng.standard_normal((K - 1, N))
        greens = np.empty((K, G), np.int64)
        fracs = np.empty((K, N), np.float64)
        offsets = np.empty((K, N), np.int64)
        greens[0], fracs[0], offsets[0] = inc_g, inc_u, inc_o
        greens[1:] = np.clip(np.rint(mg + sg * zg), space.lo, space.hi).astype(np.int64)
        fracs[1:] = np.mod(mu + su * zu, 1.0)
        for k in range(1, K):
            offsets[k] = offsets_of(space, greens[k], fracs[k])
        scores = np.asarray(objective(greens, offsets), np.float64)
        if gen == 0:
            out['shipped_score'] = float(scores[0])
        elif scores[0] != inc_score:
            raise RuntimeError('generation %d: the incumbent scored %r, not the %r it scored before; the objective is '
                               'not deterministic' % (gen, float(scores[0]), inc_score))
        order = np.argsort(-scores, kind='stable')
        elites = order[:n_elites(K, elite_frac)]
        best = int(order[0])
        inc_g, inc_u, inc_o, inc_score = greens[best].copy(), fracs[best].copy(), offsets[best].copy(), float(scores[best])
        row = dict(generation=gen, incumbent_reward=inc_score, best_reward=float(scores[best]),
                   mean_reward=float(scores.mean()), elite_mean_reward=float(scores[elites].mean()),
                   green_std=float(sg.mean()) if G else 0.0, offset_std=float(su.mean()))
        mg, sg = greens[elites].mean(axis=0), np.maximum(greens[elites].std(axis=0), GREEN_STD_FLOOR)
        mu, su = circular_mean_std(fracs[elites])
        su = np.maximum(su, OFFSET_STD_FLOOR)
        for key, v in (('greens', greens), ('offsets', offsets), ('scores', scores), ('rows', row)):
            out[key].append(v)
        if on_generation is not None:
            on_generation(row)
    out.update(best_greens=inc_g, best_offsets=inc_o, best_score=inc_score)
    return out


def check_settings(seeds, config_test_seeds, candidates, generations, elite_frac, min_green, max_green):
    """The refusals that need no env: ValueError naming the setting."""
    seeds = [int(s) for s in seeds]
    if not seeds:
        raise ValueError('tune_fixedtime: no tuning seeds')
    held = sorted(set(seeds) & (set(int(s) for s in config_test_seeds) | set(EVALUATION_SEEDS)))
    if held:
        raise ValueError('tune_fixedtime: tuning seeds %s are evaluation seeds (the config\'s test_seeds or the '
                         'evaluation scripts\' defaults %d..%d); tune on other seeds' % (held, EVALUATION_SEEDS[0],
                                                                                        EVALUATION_SEEDS[-1]))
    if int(candidates) < 2:
        raise ValueError('tune_fixedtime: candidates must be at least 2 (got %d)' % candidates)
    if not 0.0 < float(elite_frac) <= 1.0:
        raise ValueError('tune_fixedtime: elite_frac must be in (0, 1] (got %r)' % elite_frac)
    if int(min_green) < 1 or int(min_green) > int(max_green):
        raise ValueError('tune_fixedtime: need 1 <= min_green <= max_green (got %d, %d)' % (min_green, max_green))
    if int(generations) < 0:
        raise ValueError('tune_fixedtime: generations must be at least 0 (got %d)' % generations)
    return seeds


def written_programs(env, program):
    """{tlLogic id: {'offset', 'phases'}} of a SignalProgram on `env`: the states of the env's own programs, the
    durations and offsets of `program`."""
    from ..envs.fixedtime import env_programs
    own = env_programs(env)
    out = {}
    for i, name in enumerate(env._tables.node_names):
        states = [st for _, st in own[name]['phases']]
        out[name] = {'offset': int(program.offset[i]),
                     'phases': [[int(program.dur[i, k]), states[k]] for k in range(int(program.n_phases[i]))]}
    return out


class _Member:
    """A fixed-time member of the search's group: the evaluator reads `name` and `program`."""
    name = 'fixedtime'

    def __init__(self, program):
        self.program = program


def tune_fixedtime(config_path, base_dir, seeds, candidates=512, generations=30, elite_frac=0.1, min_green=5,
                   max_green=60, rng_seed=0, device=0):
    """Tune the config's fixed-time plan on `seeds` and write `<base_dir>/fixedtime/` (module docstring).  Returns
    {'greens', 'offsets', 'scores' (per generation), 'best_program', 'best_score', 'shipped_score', 'dir'}."""
    from ..envs import make_env
    from ..envs.fixedtime import env_program, write_tll
    from .evaluator import _Group
    config = configparser.ConfigParser()
    if not config.read(config_path):
        raise ValueError('tune_fixedtime: no config %s' % config_path)
    cfg = config['ENV_CONFIG']
    own_test = [s for s in cfg.get('test_seeds', '').split(',') if s.strip()]
    seeds = check_settings(seeds, own_test, candidates, generations, elite_frac, min_green, max_green)
    out_dir = os.path.join(base_dir, 'fixedtime')
    data = os.path.join(out_dir, 'data')
    tll = os.path.abspath(os.path.join(data, 'tuned.tll.xml'))
    if os.path.exists(tll):
        raise ValueError('tune_fixedtime: %s exists; tune into another directory' % tll)
    ecfg = configparser.ConfigParser()
    ecfg.read_dict(config)
    ecfg['ENV_CONFIG']['test_seeds'] = ','.join(str(s) for s in seeds)
    ecfg['ENV_CONFIG']['agent'] = 'fixedtime'
    env = make_env(ecfg['ENV_CONFIG'], len(seeds), data + os.sep, is_record=False, device=device)
    try:
        shipped = env_program(env)
    except ValueError as e:
        raise ValueError('tune_fixedtime: scenario %r has no fixed-time programs (%s)' % (env.name, e)) from None
    os.makedirs(data, exist_ok=True)
    space = search_space(shipped, min_green, max_green)
    K = int(candidates)
    members = [_Member(shipped) for _ in range(K)]
    group = _Group([env] * K, members, [env.seed] * K, ['candidate %d' % k for k in range(K)], 'default',
                   device=device)

    def objective(greens, offsets):
        for k, m in enumerate(members):
            m.program = space.program(greens[k], offsets[k])
        group.episode()
        return np.array([float(np.mean(mean)) for mean, _ in group.rewards()])

    t0 = time.time()

    def log(row):
        logging.info('generation %d: incumbent %.4f, best %.4f, mean %.4f, elite mean %.4f (%.1f s)'
                     % (row['generation'], row['incumbent_reward'], row['best_reward'], row['mean_reward'],
                        row['elite_mean_reward'], time.time() - t0))

    if int(generations) == 0:
        score = float(objective(np.repeat(space.d0[None], K, 0), np.repeat(np.asarray(shipped.offset, np.int64)[None],
                                                                              K, 0))[0])
        res = dict(greens=[], offsets=[], scores=[], rows=[], best_greens=space.d0, best_score=score,
                   best_offsets=np.asarray(shipped.offset, np.int64), shipped_score=score)
    else:
        res = cem(space, objective, K, generations, elite_frac, rng_seed, on_generation=log)
    best = space.program(res['best_greens'], res['best_offsets'])
    write_tll(written_programs(env, best), tll)
    ecfg_out = configparser.ConfigParser()
    ecfg_out.read_dict(config)
    ecfg_out['ENV_CONFIG']['tll_file'] = tll
    with open(os.path.join(data, os.path.basename(config_path)), 'w') as f:
        ecfg_out.write(f)
    cols = ('generation', 'incumbent_reward', 'best_reward', 'mean_reward', 'elite_mean_reward', 'green_std',
            'offset_std')
    with open(os.path.join(data, 'tune_log.csv'), 'w', newline='') as f:
        w = csv.writer(f)
        w.writerow(cols)
        for row in res['rows']:
            w.writerow([row[c] if c == 'generation' else repr(row[c]) for c in cols])
    names = env._tables.node_names
    info = dict(config=os.path.basename(config_path), scenario=env.name, seeds=seeds, candidates=K,
                generations=int(generations), elite_frac=float(elite_frac), min_green=int(min_green),
                max_green=int(max_green), rng_seed=int(rng_seed), elites=n_elites(K, elite_frac),
                bounds=[dict(node=names[int(i)], phase=int(k), lo=int(lo), hi=int(hi), d0=int(d))
                        for i, k, lo, hi, d in zip(space.node, space.phase, space.lo, space.hi, space.d0)],
                shipped_score=res['shipped_score'], final_score=res['best_score'])
    with open(os.path.join(data, 'tune.json'), 'w') as f:
        json.dump(info, f, indent=1)
    logging.info('tuned %s: %.4f -> %.4f in %.1f s, written to %s' % (env.name, res['shipped_score'], res['best_score'],
                                                                      time.time() - t0, out_dir))
    return dict(greens=res['greens'], offsets=res['offsets'], scores=res['scores'], best_program=best,
                best_score=res['best_score'], shipped_score=res['shipped_score'], dir=out_dir)
