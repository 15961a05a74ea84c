"""Builder of the batch wire format of include/rbgtopo.h (BLOB section)."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence, Tuple

import numpy as np

MAGIC = 0x54474252
VERSION = 1
HDR_WORDS = 8
STEP_WORDS = 16
STEP_EXCLUSIVE = 1
STEP_GANG = 2
ROLE_EXCLUSIVE = 1
MAX_STEP_ROLES = 8
MAX_STEP_REPLICAS = 32
MAX_GROUP_ROLES = 16
NEED_CAP = 16


@dataclass
class Step:
    """One wave of one dependency level of one RoleBasedGroup."""
    gid: int
    roles: List[Tuple[int, int, int, int]]          # (count, demand, need, role_flags)
    pair: Sequence[Sequence[int]] = field(default_factory=list)  # [P][Q]
    anchors: List[Tuple[int, int, int]] = field(default_factory=list)   # (node, role q, count)
    consumed: List[Tuple[int, int]] = field(default_factory=list)       # (node, amount)
    flags: int = 0
    fixed_domain: int = -1
    level: int = 0      # exclusive level (word +14; DESIGN.md §3.9)

    @property
    def n_replicas(self) -> int:
        return sum(r[0] for r in self.roles)


class BlobBuilder:
    def __init__(self) -> None:
        self.steps: List[Step] = []

    def add(self, step: Step) -> "BlobBuilder":
        self.steps.append(step)
        return self

    def build(self) -> np.ndarray:
        ns = len(self.steps)
        body: List[int] = []
        table = np.zeros((ns, STEP_WORDS), dtype=np.int64)
        base = HDR_WORDS + ns * STEP_WORDS
        racc = pacc = 0
        for i, s in enumerate(self.steps):
            P = len(s.roles)
            Q = len(s.pair[0]) if (len(s.pair) and len(s.pair[0])) else 0
            while (base + len(body)) & 3:      # role records are read as 16-byte vectors
                body.append(0)
            role_off = base + len(body)
            for r in s.roles:
                body.extend(int(x) for x in r)
            pair_off = base + len(body)
            for p in range(P):
                row = s.pair[p] if Q else []
                assert len(row) == Q
                body.extend(int(x) for x in row)
            anchor_off = base + len(body)
            for a in s.anchors:
                body.extend(int(x) for x in a)
            cons_off = base + len(body)
            for c in s.consumed:
                body.extend(int(x) for x in c)
            R = s.n_replicas
            table[i] = [s.gid, s.flags, s.fixed_domain, P, role_off, Q, pair_off, len(s.anchors),
                        anchor_off, len(s.consumed), cons_off, R, racc, pacc, s.level, 0]
            racc += R
            pacc += P
        words = base + len(body)
        out = np.zeros(words, dtype=np.int32)
        out[0:8] = [MAGIC, VERSION, ns, words, racc, pacc, 0, 0]
        out[HDR_WORDS:base] = table.reshape(-1)
        out[base:] = np.asarray(body, dtype=np.int64) if body else []
        return out


def blob_totals(blob: np.ndarray) -> Tuple[int, int, int]:
    """(n_steps, total replicas, total role rows) of a built blob."""
    return int(blob[2]), int(blob[4]), int(blob[5])


GROUPS_MAGIC = 0x47474252
GROUP_WORDS = 12


@dataclass
class Group:
    """A whole RoleBasedGroup for rbgtopo_place_groups; roles sorted by (level, name)."""
    gid: int
    roles: List[Tuple[int, int, int, int]]          # (level, pending, demand, role_flags)
    pair: Sequence[Sequence[int]]                    # [Q][Q]
    anchors: List[Tuple[int, int, int]] = field(default_factory=list)
    flags: int = 0
    fixed_domain: int = -1
    level: int = 0      # exclusive level (word +10; DESIGN.md §3.9)


class GroupsBuilder:
    def __init__(self) -> None:
        self.groups: List[Group] = []

    def add(self, g: Group) -> "GroupsBuilder":
        self.groups.append(g)
        return self

    def build(self) -> np.ndarray:
        ng = len(self.groups)
        base = HDR_WORDS + ng * GROUP_WORDS
        table = np.zeros((ng, GROUP_WORDS), dtype=np.int64)
        body: List[int] = []
        pacc = 0
        for i, g in enumerate(self.groups):
            q = len(g.roles)
            role_off = base + len(body)
            for r in g.roles:
                body.extend(int(x) for x in r)
            pair_off = base + len(body)
            for row in g.pair:
                assert len(row) == q
                body.extend(int(x) for x in row)
            anchor_off = base + len(body)
            for a in g.anchors:
                body.extend(int(x) for x in a)
            pend = sum(r[1] for r in g.roles)
            table[i] = [g.gid, g.flags, g.fixed_domain, q, role_off, pair_off, len(g.anchors), anchor_off,
                        pacc, pend, g.level, 0]
            pacc += pend
        words = base + len(body)
        out = np.zeros(words, dtype=np.int32)
        out[0:8] = [GROUPS_MAGIC, VERSION, ng, words, pacc, 0, 0, 0]
        out[HDR_WORDS:base] = table.reshape(-1)
        out[base:] = np.asarray(body, dtype=np.int64) if body else []
        return out


def tile_groups_blob(blob: np.ndarray, copies: int, gid_stride: int = 1) -> np.ndarray:
    """Replicate a 1-group blob `copies` times with gids gid0 + i*gid_stride
    (vectorised: fleets of identical shapes)."""
    assert int(blob[2]) == 1
    rec = blob[HDR_WORDS:HDR_WORDS + GROUP_WORDS].astype(np.int64)
    body = blob[HDR_WORDS + GROUP_WORDS:].astype(np.int64)
    nb = len(body)
    base = HDR_WORDS + copies * GROUP_WORDS
    table = np.tile(rec, (copies, 1))
    i = np.arange(copies, dtype=np.int64)
    shift = (base - (HDR_WORDS + GROUP_WORDS)) + i * nb
    table[:, 0] = rec[0] + i * gid_stride
    for col in (4, 5, 7):
        table[:, col] = rec[col] + shift
    table[:, 8] = i * rec[9]
    out = np.zeros(base + copies * nb, dtype=np.int32)
    out[0:8] = [GROUPS_MAGIC, VERSION, copies, len(out), copies * rec[9], 0, 0, 0]
    out[HDR_WORDS:base] = table.reshape(-1)
    out[base:] = np.tile(body, copies)
    return out
