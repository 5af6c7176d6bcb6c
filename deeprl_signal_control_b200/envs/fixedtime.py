"""Fixed-time signal control: every node runs the static signal program its net ships with, the definition the FIXED
mode of `tsc_step_kernel` computes on the device (`tsc_set_signal_program`).

Node i runs P_i phases.  Phase k lasts d_k >= 1 whole seconds and shows three link masks, bit j = character j of its
state string: open = 'G' or 'g', major = 'G', yellow = 'y' (the words node_signal produces for the action path; 'r' is
closed).  The cycle is C_i = sum of the d_k, and the simulated second s -> s + 1 runs with the phase k whose window
[start_k, start_k + d_k) holds (s - offset_i) mod C_i: as in SUMO, a positive offset delays every phase.  A control
interval records the phase in force during its first simulated second (the control CSV's action column, the phase tap
of tsc_get_counts), a function of time alone.

Programs come in the form of net.sumo_ingest.read_signal_programs, {tlLogic id: {'type', 'offset', 'phases':
[[duration, state], ...]}}: the grid's and the small grid's restate their generators' exp.tll.xml, Monaco's are read
from most.net.xml (or its cache), a SUMO-file scenario's from its net and additional files.  An [ENV_CONFIG] `tll_file`
replaces the programs of the ids its <tlLogic> elements name.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass

import numpy as np

TSC_MAX_NODE_LINKS = 32                 # include/tsc.h: link masks are uint32
_MONACO_CACHE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'net', 'data',
                             'real_net_programs.json')


@dataclass
class SignalProgram:
    """One program per node, in the env's node order: int32 n_phases [N], dur [N][max_phases], offset [N]; uint32 link
    masks open / major / yellow [N][max_phases] (padding phases are zero)."""
    n_phases: np.ndarray
    dur: np.ndarray
    open: np.ndarray
    major: np.ndarray
    yellow: np.ndarray
    offset: np.ndarray

    @property
    def max_phases(self) -> int:
        return int(self.dur.shape[1])

    @property
    def cycle(self) -> np.ndarray:
        return self.dur.sum(axis=1)


def state_masks(state: str):
    """(open, major, yellow) link masks of a state string of 'G g y r'."""
    o = m = y = 0
    for j, ch in enumerate(state):
        if ch in 'Gg':
            o |= 1 << j
        if ch == 'G':
            m |= 1 << j
        if ch == 'y':
            y |= 1 << j
    return o, m, y


def _whole(tl_id, what, value, least=None):
    try:
        v = float(value)
    except (TypeError, ValueError):
        raise ValueError('tlLogic %r: %s %r is not a number' % (tl_id, what, value)) from None
    if v != int(v):
        raise ValueError('tlLogic %r: %s %r is not a whole number of seconds' % (tl_id, what, value))
    if least is not None and v < least:
        raise ValueError('tlLogic %r: %s %r is below %d' % (tl_id, what, value, least))
    return int(v)


def program_tables(node_names, n_links, programs) -> SignalProgram:
    """The SignalProgram of `programs` ({tlLogic id: program}) on an env whose signalised nodes are `node_names`, node i
    having n_links[i] controlled links.  Refuses (ValueError naming the tlLogic id and the reason) a program that names
    no node, a node without a program, a type other than static, a state character outside 'G g y r', a duration that
    is not a whole number of seconds of at least 1, and a state whose length is not the node's link count or exceeds
    TSC_MAX_NODE_LINKS."""
    names = list(node_names)
    for tl_id in programs:
        if tl_id not in names:
            raise ValueError('tlLogic %r names no signalised node of the env' % (tl_id,))
    rows = []
    for name, nl in zip(names, n_links):
        if name not in programs:
            raise ValueError('tlLogic %r: the signalised node has no program' % (name,))
        prog = programs[name]
        if prog.get('type', 'static') != 'static':
            raise ValueError('tlLogic %r: type %r is not static (only static programs run)' % (name, prog['type']))
        if not prog['phases']:
            raise ValueError('tlLogic %r: the program has no phase' % (name,))
        offset = _whole(name, 'offset', prog.get('offset', 0))
        phases = []
        for dur, state in prog['phases']:
            bad = [ch for ch in state if ch not in 'Ggyr']
            if bad:
                raise ValueError('tlLogic %r: state %r has the character %r (only G g y r run)' % (name, state, bad[0]))
            if len(state) > TSC_MAX_NODE_LINKS:
                raise ValueError('tlLogic %r: state %r has %d links, more than TSC_MAX_NODE_LINKS = %d'
                                 % (name, state, len(state), TSC_MAX_NODE_LINKS))
            if len(state) != nl:
                raise ValueError('tlLogic %r: state %r has %d links, the node has %d' % (name, state, len(state), nl))
            phases.append((_whole(name, 'duration', dur, least=1),) + state_masks(state))
        rows.append((offset, phases))
    N, P = len(rows), max([len(p) for _, p in rows] + [1])
    out = SignalProgram(n_phases=np.zeros(N, np.int32), dur=np.zeros((N, P), np.int32), open=np.zeros((N, P), np.uint32),
                        major=np.zeros((N, P), np.uint32), yellow=np.zeros((N, P), np.uint32),
                        offset=np.zeros(N, np.int32))
    for i, (offset, phases) in enumerate(rows):
        out.n_phases[i], out.offset[i] = len(phases), offset
        for k, (d, o, m, y) in enumerate(phases):
            out.dur[i, k], out.open[i, k], out.major[i, k], out.yellow[i, k] = d, o, m, y
    return out


def phase_at(program: SignalProgram, sec: int) -> np.ndarray:
    """int32 [N]: the phase of every node in force during simulated second `sec`."""
    out = np.zeros(len(program.n_phases), np.int32)
    for i, (n_p, off) in enumerate(zip(program.n_phases, program.offset)):
        t = (int(sec) - int(off)) % int(program.dur[i, :n_p].sum())
        k = 0
        while k < n_p - 1 and t >= program.dur[i, k]:
            t -= int(program.dur[i, k])
            k += 1
        out[i] = k
    return out


def scenario_programs(env):
    """The env's programs ({tlLogic id: program}) before any `tll_file` override."""
    from ..net import sumo_ingest
    if env.name == 'large_grid':
        from ..net.large_grid import tls_programs
        return tls_programs()
    if env.name == 'small_grid':
        from ..net.small_grid import tls_programs
        return tls_programs()
    if getattr(env, 'net_file', None):                      # SUMO-file scenario (envs/sumo_env.py)
        return sumo_ingest.read_signal_programs(env.net_file, env.tll_file)
    if env.name == 'real_net':
        net_file = os.path.join(env.data_path or '', 'in', 'most.net.xml')
        if os.path.exists(net_file):
            return sumo_ingest.read_signal_programs(net_file)
        with open(_MONACO_CACHE) as f:
            return json.load(f)
    raise ValueError('no fixed-time programs for scenario %r' % env.name)


def env_programs(env):
    """The programs ({tlLogic id: program}) a scenario env runs: its scenario's, those named by its `tll_file`
    replaced."""
    from ..net import sumo_ingest
    programs = dict(scenario_programs(env))
    if env.tll_file:
        programs.update(sumo_ingest.read_signal_programs(env.tll_file))
    return programs


def env_program(env) -> SignalProgram:
    """The SignalProgram of a scenario env: its scenario's programs, those named by its `tll_file` replaced."""
    net = env._tables
    return program_tables(net.node_names, [len(net.phases[n][0]) for n in net.node_names], env_programs(env))


def program_key(program: SignalProgram):
    """Equal for two SignalPrograms with the same tables (padding included)."""
    return tuple(np.asarray(getattr(program, f)).tobytes() for f in ('n_phases', 'dur', 'open', 'major', 'yellow', 'offset'))


def write_tll(programs, path) -> str:
    """Write `programs` ({tlLogic id: {'offset', 'phases': [[duration, state], ...]}}) as a SUMO additional file of
    static programs, in the given id order: `<additional><tlLogic id type="static" programID="tuned" offset><phase
    duration state/>...`, durations and offsets as whole-second integers.  The inverse of
    net.sumo_ingest.read_signal_programs for static programs: program_tables of what it reads back gives the tables of
    `programs`.  Returns `path`."""
    from xml.sax.saxutils import quoteattr
    lines = ['<additional>']
    for tl_id, prog in programs.items():
        if prog.get('type', 'static') != 'static':
            raise ValueError('tlLogic %r: type %r is not static (only static programs are written)' % (tl_id, prog['type']))
        lines.append('    <tlLogic id=%s type="static" programID="tuned" offset="%d">'
                     % (quoteattr(str(tl_id)), _whole(tl_id, 'offset', prog.get('offset', 0))))
        for dur, state in prog['phases']:
            lines.append('        <phase duration="%d" state=%s/>' % (_whole(tl_id, 'duration', dur, least=1),
                                                                       quoteattr(str(state))))
        lines.append('    </tlLogic>')
    lines.append('</additional>')
    with open(path, 'w') as f:
        f.write('\n'.join(lines) + '\n')
    return path


class FixedTimeController:
    """Fixed-time controller with the reference controllers' one-replica protocol: `forward(obs)` ignores the
    observation and returns the program phases in force at the env's current second, the actions the env records.  The
    simulator runs the program itself (envs.fixedtime_controller sets it), so the actions passed to step are not
    read."""

    def __init__(self, env):
        self.name = 'fixedtime'
        self.env = env
        self.node_names = env.node_names
        self.program = env_program(env)

    def forward(self, obs):
        return phase_at(self.program, self.env.cur_sec)
