"""Max-pressure signal control (Varaiya 2013) in numpy: the definition `tsc_pressure_actions` computes on the device.

For replica r, node i and phase p < node_n_phases[i]:

    P(r, i, p) = sum over links l with link_node[l] == i and bit link_tlidx[l] set in node_green[i][p]
                 of lane_cnt[r][link_from[l]] - lane_cnt[r][link_to[l]]

and the action of node i is the first p with the largest P (np.argmax).  Lane counts are whole-lane vehicle counts
(the `lane_cnt` of `BatchedSim.dump_state`), so the arithmetic is integer.  Uncontrolled links (link_node = -1) do not
count, nor do links into a lane the net does not hold (link_to = -1: Monaco's connections to lanes no passenger car may
use, which no vehicle takes); permissive 'g' is green, as node_green defines it.  No minimum green and no cycle: yellow
insertion on a phase change is the environment's.
"""
from __future__ import annotations

import numpy as np


def pressure_links(net):
    """The per-node controlled links of a NetTables: (off [n_nodes + 1], from, to, tlidx), node i's links being entries
    off[i] .. off[i + 1] in link index order."""
    node = np.asarray(net.link_node, np.int64)
    keep = np.flatnonzero((node >= 0) & (np.asarray(net.link_from) >= 0) & (np.asarray(net.link_to) >= 0))
    keep = keep[np.argsort(node[keep], kind="stable")]
    off = np.searchsorted(node[keep], np.arange(net.n_nodes + 1)).astype(np.int64)
    return (off, np.asarray(net.link_from, np.int64)[keep], np.asarray(net.link_to, np.int64)[keep],
            np.asarray(net.link_tlidx, np.int64)[keep])


def pressure_actions(net, lane_cnt):
    """Max-pressure actions of lane counts `lane_cnt` [..., n_lanes]: int32 [..., n_nodes]."""
    cnt = np.asarray(lane_cnt, np.int64)
    off, fr, to, tl = pressure_links(net)
    diff = cnt[..., fr] - cnt[..., to]
    green = np.asarray(net.node_green, np.int64).reshape(net.n_nodes, -1)
    out = np.zeros(cnt.shape[:-1] + (net.n_nodes,), np.int32)
    for i in range(net.n_nodes):
        n_p, links = int(net.node_n_phases[i]), slice(off[i], off[i + 1])
        if n_p == 0:
            continue
        on = (green[i, :n_p, None] >> tl[None, links]) & 1            # [phase][link of node i]
        out[..., i] = np.argmax(diff[..., links] @ on.T, axis=-1)
    return out


class MaxPressureController:
    """Max-pressure controller with the reference controllers' one-replica protocol: `forward(obs)` ignores the
    observation and returns the actions of the env's replica 0 from its lane counts (tsc_dump_state) after the last
    reset / step.  The batched evaluators compute the same actions on the device (tsc_pressure_actions)."""

    def __init__(self, env):
        self.name = 'maxpressure'
        self.env = env
        self.node_names = env.node_names

    def forward(self, obs):
        cnt, _ = self.env._ensure_sim().dump_state(0)
        return pressure_actions(self.env._tables, cnt)
