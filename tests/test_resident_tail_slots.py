"""The global tail of the resident Arnoldi kernel, restated on the CPU: where each tail pair is copied, when it is read, and
the order of the cp.async groups and bulk copies of one thread.

At N = 100 a CTA of `resident3g_arnoldi_kernel` (csrc/gmres.cu) owns 15 152 rows, 30 row pairs per thread; the two
shared-memory stages hold the first qs of them and the pairs q >= qs (the global tail) travel by 16-byte cp.async into stage
slots the thread has released:
  * update sweep of a shared-memory-role v_t: after pair R3_TAIL_AT - 1 the pairs qs .. qs + R3_TAIL_AT - 1 are copied into
    slots 0 .. R3_TAIL_AT - 1 of v_t's own stage (only when qs >= R3_TAIL_AT), and applied last;
  * dot sweep of v_{t+1} when it is stage 0's (step t = 2 mod 3): the pairs qs .. 2 qs - 1, copied at the end of step t - 1
    into slots 0 .. qs - 1 of stage 1, whose refill with v_{t+2} moves behind the barrier after that dot sweep.
`Thread` below replays one thread's accesses in program order over a whole Arnoldi step and checks, for every split
qs = 1 .. 30 and the N = 100, N = 80 and 2D row geometries (first, last and empty CTAs, every kind of thread):
  1. every read of a stage slot finds the pair it expects, completed (so no copy overwrote a slot before its last read, and
     no copy or bulk copy was still in flight), and no copy targets a stage a bulk copy is filling;
  2. every copy source lies in this CTA's rows of one species' segment of the vector, 16-byte aligned, and every slot inside
     its stage;
  3. a bulk copy into a stage follows this thread's fence.proxy.async and the CTA barrier;
  4. the groups pending at each cp.async.wait_group are the documented ones, and never more than two.
The kernel's constants are read from the source, so a change there that this restatement does not follow fails here.
"""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "nonlinearsolve.jl_b200", "csrc", "gmres.cu")).read()


def _const(name):
    m = re.search(r"constexpr\s+int\s+%s\s*=\s*(\d+)\s*;" % name, SRC)
    assert m, "constant %s not found in gmres.cu" % name
    return int(m.group(1))


R3_THREADS, R3_RP, R3_RPR, R3_TAIL_AT = (_const(n) for n in ("R3_THREADS", "R3_RP", "R3_RPR", "R3_TAIL_AT"))
PAIR = 2 * R3_THREADS
ANNEX_BYTES = (R3_RP - R3_RPR) * R3_THREADS * 16
G_H100, SMEM_H100 = 132, 232448


def test_constants_and_slot_rules_match_the_source():
    assert (R3_THREADS, R3_RP, R3_RPR, R3_TAIL_AT) == (256, 30, 16, 9)
    assert "constexpr size_t R3_ANNEX_BYTES = (size_t)(R3_RP - R3_RPR) * R3_THREADS * 16;" in SRC
    assert "return cx.qs > q / 2; }  // q < 2 qs" in SRC                                   # dot-sweep slots
    assert "return cx.qs >= R3_TAIL_AT && cx.qs > q - R3_TAIL_AT; }" in SRC                # update-sweep slots
    assert SRC.count("r3_tail_copy(cx, vcur, sc, R3_TAIL_AT, lim, lims, hop)") == 2      # both update sweeps, after pair R3_TAIL_AT - 1
    assert SRC.count("q + 1 == R3_TAIL_AT && cx.qs >= R3_TAIL_AT && tail") == 2
    assert "sc, cx.qs, lim, lims, hop)" in SRC                                              # the dot-sweep tail: qs slots


def plan_qs(n_cells, G, smem, cap=None):
    cpc = -(-n_cells // G)
    cpc += cpc & 1
    spare = smem - ANNEX_BYTES - 2048
    qs = min(R3_RP, -(-2 * cpc // PAIR), spare // (2 * 8 * PAIR))
    return cpc, (qs if cap is None else min(qs, cap))


def update_slot(qs, q):
    return qs >= R3_TAIL_AT and qs > q - R3_TAIL_AT


def dot_slot(qs, q):
    return qs > q // 2


class Violation(AssertionError):
    pass


class Thread:
    """One thread `tid` of CTA b: its accesses to the stages, in program order, over one Arnoldi step of `total` sweeps."""

    def __init__(self, n_cells, cpc, b, tid, qs, total):
        self.NC, self.cpc, self.b, self.tid, self.qs, self.total = n_cells, cpc, b, tid, qs, total
        self.ncell = max(0, min(cpc, n_cells - b * cpc))
        self.nrow = 2 * self.ncell
        self.lim, self.lims = self.nrow - 2 * tid, self.ncell - 2 * tid
        self.hop = n_cells - self.ncell
        self.sw = min(2 * cpc, PAIR * qs)
        self.defer = self.nrow > PAIR * qs
        self.tail = self.lim > PAIR * qs
        # stage s, slot j -> (vector, pair, complete?); bulk copy in flight per stage; pending cp.async groups
        self.slot = [dict(), dict()]
        self.tma = [None, None]
        self.groups = []
        self.fenced = False
        self.wait_log = []
        self.copies = 0

    def copies_into(self, stage):
        """slots of `stage` this thread has written by cp.async since the last bulk copy into it"""
        return [j for j, (v, q, _) in self.slot[stage].items() if q >= self.qs]

    def exists(self, q):
        return PAIR * q < self.lim

    def fail(self, msg):
        raise Violation("CTA %d tid %d qs %d: %s" % (self.b, self.tid, self.qs, msg))

    # ---- primitives
    def bulk(self, stage, v):                         # thread 0 after the barrier; every thread checks its own slots
        if not self.fenced:
            self.fail("bulk copy into stage %d without fence.proxy.async + barrier" % stage)
        for j, (_, _, done) in self.slot[stage].items():
            if not done:
                self.fail("bulk copy into stage %d over an incomplete cp.async (slot %d)" % (stage, j))
        if self.tma[stage] is not None:
            self.fail("two bulk copies in flight into stage %d" % stage)
        self.tma[stage] = v
        self.fenced = False
        self.slot[stage] = {}

    def mbar_wait(self, stage, v):
        if self.tma[stage] != v:
            self.fail("waited for v%d in stage %d, in flight: %s" % (v, stage, self.tma[stage]))
        self.tma[stage] = None
        for q in range(min(self.qs, R3_RP)):          # the staged prefix: pair q in slot q
            if PAIR * q + 2 * self.tid < self.sw:
                self.slot[stage][q] = (v, q, True)

    def copy(self, stage, v, pairs, kind):
        """one group: pairs[i] -> slot i"""
        if self.tma[stage] is not None:
            self.fail("cp.async into stage %d while a bulk copy fills it" % stage)
        writes = []
        for j, q in enumerate(pairs):
            lr = PAIR * q
            if lr >= self.lim:
                break
            src = 2 * self.tid + lr + (self.hop if lr >= self.lims else 0)   # relative to the CTA's first cell
            e = self.b * self.cpc + src
            seg0 = (self.b * self.cpc, self.b * self.cpc + self.ncell)
            seg1 = (self.NC + seg0[0], self.NC + seg0[1])
            if not (seg0[0] <= e and e + 1 < seg0[1] or seg1[0] <= e and e + 1 < seg1[1]):
                self.fail("source element %d of pair %d outside this CTA's rows" % (e, q))
            if e % 2 or not 0 <= e < 2 * self.NC - 1:
                self.fail("source element %d misaligned or outside the vector" % e)
            off = PAIR * j + 2 * self.tid
            if off + 1 >= self.sw:
                self.fail("slot %d (offset %d) outside stage of %d doubles" % (j, off, self.sw))
            self.slot[stage][j] = (v, q, False)
            writes.append((stage, j))
            self.copies += 1
        self.groups.append((kind, writes))

    def wait_all(self, where):
        self.wait_log.append((where, tuple(k for k, _ in self.groups)))
        for _, writes in self.groups:
            for stage, j in writes:
                v, q, _ = self.slot[stage][j]
                self.slot[stage][j] = (v, q, True)
        self.groups = []

    def read(self, stage, j, v, q):
        got = self.slot[stage].get(j)
        if got != (v, q, True):
            self.fail("pair %d of v%d: slot %d of stage %d holds %s" % (q, v, j, stage, got))

    # ---- one sweep over the pairs of an smem-role vector
    def sweep(self, stage, v, slot_stage, slot_rule, issue=None):
        for q in range(R3_RP):
            if self.exists(q):
                if q < self.qs:
                    self.read(stage, q, v, q)
                elif slot_rule(self.qs, q):
                    if q == self.qs:
                        self.wait_all("sweep v%d" % v)
                    self.read(slot_stage, q - self.qs, v, q)
                # else: straight from global memory
            if issue is not None and q + 1 == R3_TAIL_AT and self.qs >= R3_TAIL_AT and self.tail:
                self.copy(stage, v, range(self.qs, self.qs + R3_TAIL_AT), "update")

    def run(self):
        T, qs = self.total, self.qs
        for v in range(min(T, 2) if self.nrow > 0 else 0):   # the first two vectors (nothing touched the stages before)
            self.fenced = True
            self.bulk(v, v)
        if T > 2:
            self.groups.append(("regs", []))           # register stage of v2 (its annex is not a stage)
        if self.nrow > 0:
            self.mbar_wait(0, 0)
        self.sweep(0, 0, None, lambda qs, q: False)   # prologue dot sweep of v0: tail from global memory
        for t in range(T):
            role, nxt = t % 3, (t + 1) % 3
            more = t + 1 < T
            if more:
                if nxt != 2 and self.nrow > 0:
                    self.mbar_wait(nxt, t + 1)
                if nxt == 2:
                    self.wait_all("register stage v%d" % (t + 1))
                elif nxt == 0:
                    self.sweep(0, t + 1, 1, dot_slot)
                else:
                    self.sweep(1, t + 1, None, lambda qs, q: False)
            if role == 2 and self.tail:
                self.fenced = True                     # fence.proxy.async (threads that wrote by cp.async), then the barrier
            elif role == 2 and self.defer:
                self.fenced = not any(self.copies_into(1))
            if role == 2 and self.defer and t + 2 < T and self.nrow > 0:
                self.bulk(1, t + 2)
            if role != 2:
                self.sweep(role, t, role, update_slot, issue=True)
            if role == 0 or (role == 1 and not self.defer):
                if t + 3 < T:
                    self.fenced = self.tail or not any(self.copies_into(role))
                    if self.nrow > 0:
                        self.bulk(role, t + 3)
            elif role == 1:
                if t + 2 < T and self.tail:
                    self.copy(1, t + 2, range(qs, 2 * qs), "dot")
            elif t + 3 < T:
                self.groups.append(("regs", []))
            if len(self.groups) > 2:
                self.fail("%d cp.async groups pending" % len(self.groups))
        if self.groups or any(x is not None for x in self.tma):
            self.fail("copies left in flight at the end: %s %s" % (self.groups, self.tma))


def _thread_kinds(n_cells, cpc, b):
    """Representative threads of CTA b: the first and last of each (pairs, species-boundary pair) class."""
    ncell = max(0, min(cpc, n_cells - b * cpc))
    kinds = {}
    for tid in range(R3_THREADS):
        lim, lims = 2 * ncell - 2 * tid, ncell - 2 * tid
        key = (sum(PAIR * q < lim for q in range(R3_RP)), sum(PAIR * q < lims for q in range(R3_RP)))
        kinds.setdefault(key, []).append(tid)
    return sorted({t for v in kinds.values() for t in (v[0], v[-1])})


REGIMES = {"3D N=100": 100 ** 3, "3D N=80": 80 ** 3, "2D N=1006": 1006 ** 2, "3D N=16 (empty CTAs)": 16 ** 3}


@pytest.mark.parametrize("regime", list(REGIMES))
def test_every_split_keeps_the_invariants(regime):
    n_cells = REGIMES[regime]
    cpc, qs0 = plan_qs(n_cells, G_H100, SMEM_H100)
    ctas = sorted({0, G_H100 - 1} | {b for b in range(G_H100) if b * cpc < n_cells <= (b + 1) * cpc} | ({n_cells // cpc + 1} if n_cells // cpc + 1 < G_H100 else set()))
    copies = 0
    for cap in range(1, R3_RP + 1):
        _, qs = plan_qs(n_cells, G_H100, SMEM_H100, cap)
        for b in ctas:
            for tid in _thread_kinds(n_cells, cpc, b):
                for total in (1, 2, 3, 4, 5, 6, 8, 11):
                    th = Thread(n_cells, cpc, b, tid, qs, total)
                    th.run()
                    copies += th.copies
                    for where, pending in th.wait_log:            # invariant 4: the documented groups, nothing else
                        if where.startswith("register stage"):
                            assert set(pending) <= {"regs"}, (where, pending)
                        elif pending and pending[-1] == "dot":
                            assert pending == ("dot",), (where, pending)
                        else:
                            assert set(pending) <= {"regs", "update"} and len(pending) <= 2, (where, pending)
    if regime in ("3D N=100", "2D N=1006"):
        assert copies > 0                                   # the tail exists there, and the slots are used
    else:
        assert copies == 0 or qs0 < R3_RP


def test_n100_stock_split_has_every_tail_pair_in_a_slot():
    n_cells = 100 ** 3
    cpc, qs = plan_qs(n_cells, G_H100, SMEM_H100)
    assert (cpc, qs) == (7576, 21)
    for b, tid in ((0, 0), (0, 151), (0, 152), (0, 255), (G_H100 - 1, 0), (G_H100 - 1, 255)):
        th = Thread(n_cells, cpc, b, tid, qs, 8)
        tail = [q for q in range(qs, R3_RP) if th.exists(q)]
        assert len(tail) in (8, 9), (b, tid, tail)               # 30 or 29 pairs per thread (7544 cells in the last CTA)
        assert all(update_slot(qs, q) and dot_slot(qs, q) for q in tail)
        th.run()


def test_the_model_catches_a_copy_before_the_last_read():
    """A copy issued one pair too early overwrites a slot the sweep still reads: the restatement must say so."""
    n_cells = 100 ** 3
    cpc, qs = plan_qs(n_cells, G_H100, SMEM_H100)

    class Early(Thread):
        def sweep(self, stage, v, slot_stage, slot_rule, issue=None):
            if issue is not None and self.tail and self.qs >= R3_TAIL_AT:
                self.copy(stage, v, range(self.qs, self.qs + R3_TAIL_AT), "update")
                issue = None
            for q in range(R3_RP):
                if self.exists(q):
                    if q < self.qs:
                        self.read(stage, q, v, q)
                    elif slot_rule(self.qs, q):
                        if q == self.qs:
                            self.wait_all("sweep")
                        self.read(slot_stage, q - self.qs, v, q)

    with pytest.raises(Violation, match="slot 0 of stage 0"):
        Early(n_cells, cpc, 0, 0, qs, 8).run()
