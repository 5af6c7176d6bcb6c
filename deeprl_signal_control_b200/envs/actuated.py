"""Vehicle-actuated signal control: gap-out control on per-lane induction loops, the definition the ACTUATED mode of
`tsc_step_kernel` computes on the device (`tsc_set_actuated_program`).  It restates SUMO's documented `type="actuated"`
logic; it is not pinned against SUMO.

Program.  Node i runs P_i phases in order.  Phase k shows the link masks of envs.fixedtime.state_masks (open 'G' or
'g', major 'G', yellow 'y') and lasts between minDur_k and maxDur_k whole seconds (1 <= minDur_k <= maxDur_k).  A phase
with minDur == maxDur is fixed and lasts that long; one with minDur < maxDur is actuated.

SUMO attributes.  A `type="actuated"` tlLogic takes them as SUMO documents them: minDur defaults to duration; maxDur to
duration when minDur is absent and to unbounded otherwise, represented as UNBOUNDED = 2^30 s.  A `static` program in an
`actuated` directory is converted: every phase with an open link that carries a loop and no yellow link gets minDur = 5,
maxDur = 50 (the values netconvert documents for --tls.min-dur / --tls.max-dur, not checked against a netconvert here),
every other phase is fixed at its duration.  (A phase none of whose open links the net holds has no loop to extend it;
Monaco has such phases, on links into lanes no passenger car may use, and they keep their static duration.)  The [ENV_CONFIG] keys `actuated_min_dur` / `actuated_max_dur` replace 5 / 50.

Loops.  Every lane that is the from-lane of a controlled link carries one induction loop at
X_l = max(0, len_l - detector_gap * vmax_l) from the lane start, quantised to the simulator's 1/64-m position unit
(floor), the same integer on the device and in the oracle.  detector_gap (default 2.0 s) and max_gap (default 3.0 s)
are per node, from the tlLogic's <param key="detector-gap"|"max-gap">, else from the [ENV_CONFIG] keys
`actuated_detector_gap` / `actuated_max_gap`, else the defaults.

Detection.  During second s, a vehicle on lane l whose stored front position is xq before its move and xnq after it
(1/64 m; a head vehicle that crosses or arrives has xnq = +inf) covers the loop iff xq - Lq <= X_l <= xnq, Lq =
veh_len in 1/64 m: a vehicle standing over the loop covers it.  Each lane keeps a saturating gap_l: after each second it
is 0 if a vehicle covered the loop, else min(gap_l + 1, 255); 255 after reset.  Vehicles inserted or transferred onto
the lane during second s are seen from second s + 1 on.

Decision.  At the end of second s, node i in phase k with elapsed e (the seconds k has run, s included) advances to
k + 1 mod P_i when e >= maxDur_k, or when e >= minDur_k and every controlled link open in k has gap >= max_gap_i on
its from-lane (so a phase with no such link ends at minDur).  gap counts whole seconds, so the device compares it with ceil(max_gap_i).  After an advance elapsed
restarts at 0; the resulting phase governs second s + 1.

Initial state (after every reset): the phase and elapsed time envs.fixedtime.phase_at gives for second 0 from the
durations and the offset (phase 0, elapsed 0 with offset 0).

Recorded action: the phase in force during each control interval's first second (control CSV, phase tap).

Refusals (ValueError naming the tlLogic id and the reason): everything envs.fixedtime.program_tables refuses except the
type `actuated`; types other than static and actuated; minDur > maxDur; non-whole, non-finite or zero durations,
and a duration or minDur above 2^30 s (a larger maxDur is unbounded); the phase attributes next, earliestEnd,
latestEnd, vehext, yellow and red; any <param> other than max-gap, detector-gap and the output-only show-detectors,
file and freq; max_gap <= 0 and detector_gap < 0.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

from .fixedtime import program_tables, scenario_programs

UNBOUNDED = 1 << 30
DEFAULTS = {'actuated_min_dur': 5.0, 'actuated_max_dur': 50.0, 'actuated_max_gap': 3.0, 'actuated_detector_gap': 2.0}
CONFIG_KEYS = tuple(DEFAULTS)
_REFUSED_PHASE_ATTRS = ('next', 'earliestEnd', 'latestEnd', 'vehext', 'yellow', 'red')
_PARAMS = ('max-gap', 'detector-gap', 'show-detectors', 'file', 'freq')


@dataclass
class ActuatedProgram:
    """One program per node, in the env's node order: int32 n_phases [N], min_dur / max_dur / dur [N][max_phases]
    (dur = SUMO's duration, which sets the initial state), offset [N], max_gap [N] (whole seconds, ceil of the
    seconds), init [N][2] (phase, elapsed at second 0); float64 max_gap_s / detector_gap [N] (seconds); uint32 open /
    major / yellow [N][max_phases]; int32 loop_pos [n_lanes] (1/64 m, -1 = no loop).  Padding phases are zero."""
    n_phases: np.ndarray
    min_dur: np.ndarray
    max_dur: np.ndarray
    dur: np.ndarray
    open: np.ndarray
    major: np.ndarray
    yellow: np.ndarray
    offset: np.ndarray
    max_gap: np.ndarray
    max_gap_s: np.ndarray
    detector_gap: np.ndarray
    loop_pos: np.ndarray
    init: np.ndarray

    @property
    def max_phases(self) -> int:
        return int(self.dur.shape[1])

    def key(self):
        """Bytes of every table the simulator runs: two entries share a simulator only when these are equal."""
        return tuple(np.ascontiguousarray(getattr(self, f)).tobytes()
                     for f in ('n_phases', 'min_dur', 'max_dur', 'open', 'major', 'yellow', 'max_gap', 'loop_pos', 'init'))


def config_overrides(config) -> dict:
    """The actuated [ENV_CONFIG] keys a config section sets, as floats."""
    return {k: config.getfloat(k) for k in CONFIG_KEYS if k in config}


def _seconds(tl_id, what, value, least, most=UNBOUNDED):
    """A whole number of seconds in [least, most]; `most` None: no upper bound (the caller clamps)."""
    try:
        v = float(value)
    except (TypeError, ValueError):
        raise ValueError('tlLogic %r: %s %r is not a number' % (tl_id, what, value)) from None
    if not math.isfinite(v):
        raise ValueError('tlLogic %r: %s %r is not a finite number' % (tl_id, what, value))
    if v != int(v):
        raise ValueError('tlLogic %r: %s %r is not a whole number of seconds' % (tl_id, what, value))
    if v < least:
        raise ValueError('tlLogic %r: %s %r is below %d' % (tl_id, what, value, least))
    if most is not None and v > most:
        raise ValueError('tlLogic %r: %s %r is above 2^30 s' % (tl_id, what, value))
    return int(v)


def _gap(tl_id, key, value, positive):
    try:
        v = float(value)
    except (TypeError, ValueError):
        raise ValueError('tlLogic %r: %s %r is not a number' % (tl_id, key, value)) from None
    if (positive and not v > 0) or (not positive and not v >= 0) or math.isinf(v):
        raise ValueError('tlLogic %r: %s %r must be %s' % (tl_id, key, value, 'above 0' if positive else 'at least 0'))
    return v


def phase_durations(tl_id, prog, min_dur=5, max_dur=50, loop_links=None):
    """[(minDur, maxDur)] of every phase of `prog` (the net.sumo_ingest.read_signal_programs form); `loop_links` is
    the set of the node's link indices that carry a loop (None: every link)."""
    typ = prog.get('type', 'static')
    if typ not in ('static', 'actuated'):
        raise ValueError('tlLogic %r: type %r is neither static nor actuated' % (tl_id, typ))
    attrs = prog.get('phase_attrs') or [{} for _ in prog['phases']]
    out = []
    for (dur, state), at in zip(prog['phases'], attrs):
        for a in _REFUSED_PHASE_ATTRS:
            if a in at:
                raise ValueError('tlLogic %r: the phase attribute %r is not supported' % (tl_id, a))
        d = _seconds(tl_id, 'duration', dur, 1)
        if typ == 'static':
            lo = hi = d
            if 'y' not in state and any(ch in 'Gg' and (loop_links is None or j in loop_links)
                                        for j, ch in enumerate(state)):
                lo, hi = min_dur, max_dur
        else:
            lo = _seconds(tl_id, 'minDur', at['minDur'], 1) if 'minDur' in at else d
            if 'maxDur' in at:
                hi = _seconds(tl_id, 'maxDur', at['maxDur'], 1, most=None)    # above 2^30: unbounded
            else:
                hi = d if 'minDur' not in at else UNBOUNDED
        if lo > hi:
            raise ValueError('tlLogic %r: minDur %d is above maxDur %d' % (tl_id, lo, hi))
        out.append((lo, min(hi, UNBOUNDED)))
    return out


def loop_positions(net, detector_gap) -> np.ndarray:
    """int32 [n_lanes]: X_l in 1/64 m for every from-lane of a controlled link (detector_gap of the link's node), -1
    elsewhere."""
    pos = np.full(len(net.lane_len), -1, np.int32)
    for frm, node in zip(np.asarray(net.link_from), np.asarray(net.link_node)):
        if frm < 0 or node < 0:
            continue
        x = max(0.0, float(net.lane_len[frm]) - float(detector_gap[node]) * float(net.lane_vmax[frm]))
        pos[frm] = int(math.floor(x * 64.0))
    return pos


def initial_state(dur, n_phases, offset) -> np.ndarray:
    """int32 [N][2]: the phase and elapsed seconds phase_at gives for second 0."""
    out = np.zeros((len(n_phases), 2), np.int32)
    for i, (n_p, off) in enumerate(zip(n_phases, offset)):
        t = (-int(off)) % int(dur[i, :n_p].sum())
        k = 0
        while k < n_p - 1 and t >= dur[i, k]:
            t -= int(dur[i, k])
            k += 1
        out[i] = k, t
    return out


def actuated_tables(net, programs, overrides=None) -> ActuatedProgram:
    """The ActuatedProgram of `programs` ({tlLogic id: program}) on the net tables `net` (node order, lanes, links),
    with the [ENV_CONFIG] `overrides` (config_overrides) of the defaults."""
    cfg = dict(DEFAULTS)
    cfg.update(overrides or {})
    min_d = _seconds('[ENV_CONFIG]', 'actuated_min_dur', cfg['actuated_min_dur'], 1)
    max_d = _seconds('[ENV_CONFIG]', 'actuated_max_dur', cfg['actuated_max_dur'], 1)
    if min_d > max_d:
        raise ValueError('[ENV_CONFIG]: actuated_min_dur %d is above actuated_max_dur %d' % (min_d, max_d))
    names = list(net.node_names)
    static = {k: dict(v, type='static') for k, v in programs.items()}
    base = program_tables(names, [len(net.phases[n][0]) for n in names], static)
    N, P = base.dur.shape
    lo, hi = np.zeros((N, P), np.int32), np.zeros((N, P), np.int32)
    mg_s, dg = np.zeros(N), np.zeros(N)
    loop_links = [set() for _ in names]
    for frm, node, tl in zip(np.asarray(net.link_from), np.asarray(net.link_node), np.asarray(net.link_tlidx)):
        if frm >= 0 and node >= 0:
            loop_links[node].add(int(tl))
    for i, name in enumerate(names):
        prog = programs[name]
        for k, (a, b) in enumerate(phase_durations(name, prog, min_d, max_d, loop_links[i])):
            lo[i, k], hi[i, k] = a, b
        params = prog.get('params') or {}
        for key in params:
            if key not in _PARAMS:
                raise ValueError('tlLogic %r: the <param> %r is not supported' % (name, key))
        mg_s[i] = _gap(name, 'max-gap', params.get('max-gap', cfg['actuated_max_gap']), True)
        dg[i] = _gap(name, 'detector-gap', params.get('detector-gap', cfg['actuated_detector_gap']), False)
    return ActuatedProgram(n_phases=base.n_phases, min_dur=lo, max_dur=hi, dur=base.dur, open=base.open,
                           major=base.major, yellow=base.yellow, offset=base.offset,
                           max_gap=np.array([min(math.ceil(g), 256) for g in mg_s], np.int32), max_gap_s=mg_s,
                           detector_gap=dg, loop_pos=loop_positions(net, dg),
                           init=initial_state(base.dur, base.n_phases, base.offset))


def env_program(env) -> ActuatedProgram:
    """The ActuatedProgram of a scenario env: its scenario's programs, those its `tll_file` names replaced, with the
    env's actuated [ENV_CONFIG] keys."""
    from ..net import sumo_ingest
    programs = dict(scenario_programs(env))
    if env.tll_file:
        programs.update(sumo_ingest.read_signal_programs(env.tll_file))
    return actuated_tables(env._tables, programs, getattr(env, 'actuated_cfg', None))


def fixed_program(program: ActuatedProgram):
    """The envs.fixedtime.SignalProgram a program whose phases are all fixed (min_dur == max_dur) runs as: durations
    = max_dur, offset chosen so that phase_at reproduces the initial state."""
    from .fixedtime import SignalProgram
    if not np.array_equal(program.min_dur, program.max_dur):
        raise ValueError('fixed_program: the program has actuated phases')
    off = np.zeros(len(program.n_phases), np.int32)
    for i, (k, e) in enumerate(program.init):
        off[i] = -(int(program.max_dur[i, :k].sum()) + int(e))
    return SignalProgram(n_phases=program.n_phases, dur=program.max_dur.copy(), open=program.open, major=program.major,
                         yellow=program.yellow, offset=off)


class ActuatedController:
    """Actuated controller with the reference controllers' one-replica protocol: `forward(obs)` ignores the
    observation and returns the phases the simulator's nodes show in the next simulated second
    (`tsc_get_program_phase`), the actions the env records.  The simulator runs the program itself
    (envs.actuated_controller sets it), so the actions passed to step are not read."""

    def __init__(self, env):
        self.name = 'actuated'
        self.env = env
        self.node_names = env.node_names
        self.program = env_program(env)

    def forward(self, obs):
        return self.env._ensure_sim().program_phase()[0].cpu().numpy()

