"""Oracle of ranked placement (DESIGN.md §3.10).  TEST INFRASTRUCTURE, built only on the oracle package
(oracle/wave_loop.py, oracle/placer.py): it never imports rbg_b200.

`run_fleet_ranked(topo, groups, n_alt)` runs the oracle's own level / wave loop (`wave_loop.run_fleet` with the dense
matrix of every wave), keeps the row of every replica's wave (replicas of one role in one wave share it), and then
applies §3.10 in numpy: the candidates of placed replica r are the nodes n with S_r[n] != -inf, n != assign[r],
free[n] - used_g[n] >= demand (used_g: what the group's placed replicas take on n) and, for a participating role of an
exclusive group, domain[n] == the group's reported domain; they are ranked by score descending, node ascending."""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np

from oracle import wave_loop


def _key(g: wave_loop.OGroup, ri: int, ordinal: int) -> str:
    return f"{g.name}-{g.roles[ri].name}-{ordinal}"


def run_fleet_ranked(topo, groups: Sequence[wave_loop.OGroup], n_alt: int):
    """(assign, status, domain, score[R], alt_node[R, n_alt], alt_score[R, n_alt]) in GROUPS-blob order."""
    rows: Dict[str, np.ndarray] = {}

    def on_wave(w, active, blob, r):
        off = 0
        for s in active:
            for ri, ordinal, cnt in s.waves[w]:
                row = np.array(r["matrix"][off], dtype=np.float32, copy=True)
                for c in range(cnt):
                    rows[_key(s.g, ri, ordinal + c)] = row
                off += cnt

    states, _ = wave_loop.run_fleet(topo, groups, want_matrix=True, on_wave=on_wave)
    free = np.asarray(topo.free, dtype=np.int64)
    domain = np.asarray(topo.domain, dtype=np.int64)
    assign: List[int] = []
    status, dom_out = [], []
    score: List[float] = []
    alt_node: List[List[int]] = []
    alt_score: List[List[float]] = []
    for s in states:
        res = s.result()
        status.append(res["status"])
        dom_out.append(res["domain"])
        used = np.zeros(len(free), dtype=np.int64)
        for ri in s.order:
            for c in range(s.pending[ri]):
                node = res["nodes"][_key(s.g, ri, s.first[ri] + c)]
                if node >= 0:
                    used[node] += s.g.roles[ri].demand
        for ri in s.order:
            role = s.g.roles[ri]
            for c in range(s.pending[ri]):
                node = res["nodes"][_key(s.g, ri, s.first[ri] + c)]
                assign.append(node)
                if node < 0:   # unplaced, or a failed gang
                    score.append(-np.inf)
                    alt_node.append([-1] * n_alt)
                    alt_score.append([-np.inf] * n_alt)
                    continue
                S = rows[_key(s.g, ri, s.first[ri] + c)]
                ok = (S != -np.inf) & (free - used >= role.demand)
                ok[node] = False
                if s.g.exclusive and role.exclusive:
                    ok &= domain == res["domain"]
                idx = np.nonzero(ok)[0]
                best = idx[np.lexsort((idx, -S[idx].astype(np.float64)))][:n_alt]
                score.append(float(S[node]))
                alt_node.append([int(x) for x in best] + [-1] * (n_alt - len(best)))
                alt_score.append([float(S[x]) for x in best] + [-np.inf] * (n_alt - len(best)))
    R = len(assign)
    return (np.asarray(assign, dtype=np.int32), np.asarray(status, dtype=np.int32), np.asarray(dom_out, dtype=np.int32),
            np.asarray(score, dtype=np.float32), np.asarray(alt_node, dtype=np.int32).reshape(R, n_alt),
            np.asarray(alt_score, dtype=np.float32).reshape(R, n_alt))
