"""Gangs inside network domains (kgpu_place_batch_gang_domain, kgpu_place_batch_gang_levels) and domain preemption plans
(kgpu_preempt_plan_gang_domain) under every link-weight table of test_weight_tables, and with node ids at the top of the
32-bit range.

Under the default table a member costs at most 28 * 64, so the limits these paths rely on are never approached: the
17-bit cost field of the plan node key, the 32-bit summed gang cost C_d of a trial, and K3's tile composite
cost << 15 that the commit refreshes.  Under the zero table every trial ties on cost, so the domain id decides alone.

CPU: the twins against the W-aware brute forces of test_gang_domain, test_gang_domain_levels and
test_preempt_plan_domain, and those against a plain Python reference that ranks whole tuples (a member (cost, node id,
S), a placement trial (C_d, d), a plan trial (L_d, V_d, C_d, d)) built on test_weight_tables.ref_place and ref_preempt;
the emulated kernels on the named cases of the three files (the hand-made ones under every table, the generated ones
under one table each); the domain-id tie; a summed cost past 2^31 against the arithmetic.  GPU: the device paths through
Scorer against the twins per table, on a live handle whose table changes between calls, and the summed cost past 2^31."""
import time

import numpy as np
import pytest

import test_gang_domain as GD
import test_gang_domain_levels as GL
import test_preempt_plan_domain as PD
from kubegpu_b200 import synth
from test_gang_domain import emu as place_emu, twin as place_twin                # noqa: F401  (fixtures)
from test_gang_domain_levels import emu as levels_emu, twin as levels_twin      # noqa: F401  (fixtures)
from test_preempt_plan_domain import emu as plan_emu, plans                     # noqa: F401  (fixtures)
from test_weight_tables import LIVE_ORDER, NAMES, W_of, check_reached, edge_matrix, ref_place, ref_preempt

NO_FIT = np.uint64(0xFFFFFFFFFFFFFFFF)
REQ, PREF = 1, 2
WIDE = ("flat_max", "general_edge", "one_level")           # the tables under which the edge node's k = 8 cost needs 17 bits
EDGE = 1                                                    # the index the edge node is inserted at
EDGE_MEM = 2 * max(synth.GPU_MEM_CLASSES_MIB)               # its GPU memory: only it holds a pod that needs EDGE_NEED
EDGE_NEED = max(synth.GPU_MEM_CLASSES_MIB) + 1


def top_base(N):
    return 2**32 - 1 - N


def as_tuples(keys):
    """Packed keys as (cost, node id, S), None for NO_FIT."""
    return [None if k == NO_FIT else (int(k) >> 40, int(k) >> 8 & 0xFFFFFFFF, int(k) & 0xFF) for k in keys]


def all_runs(gang):
    """[(first, end)] of every run: a gang's members, or one pod on its own."""
    out, p = [], 0
    while p < len(gang):
        e = p + 1
        while gang[p] != 0 and e < len(gang) and gang[e] == gang[p]:
            e += 1
        out.append((p, e))
        p = e
    return out


# ---- the plain Python reference ---------------------------------------------------------------------------------------
def ref_domain_place(topo, free, pods, gang, gd, dom, W, gl=None, mem=None, base=0):
    """Placement with domain levels dom[L, N] (one row: kgpu_place_batch_gang_domain), ranked on tuples.  Run by run on
    the running masks.  A constrained gang tries the levels 0 .. gang_level in order; on a level each domain d is a
    trial, ref_place of the members all or nothing on d's nodes alone, scored (C_d, d) with C_d the sum of the members'
    costs; the first level with a trial takes its smallest.  With none, REQUIRED leaves the gang out and PREFERRED is
    ref_place over every node, as is a run without a constraint.  Returns ([(cost, node id, S) or None], masks after)."""
    dom = np.atleast_2d(dom)
    F = np.array(free, np.int32)
    out = [None] * len(pods)

    def trial(nodes, p, e):
        keys, f = ref_place(topo[nodes], F[nodes], pods[p:e], W, gang=np.ones(e - p, np.int32), mem=None if mem is None else mem[nodes])
        if (keys == NO_FIT).any():
            return None
        return [(c, base + int(nodes[n]), S) for c, n, S in as_tuples(keys)], f

    for p, e in all_runs(gang):
        res = None
        if gd[p] != 0:
            for lv in range(1 + (0 if gl is None else int(gl[p]))):
                trials = []
                for d in sorted(set(dom[lv].tolist()) - {-1}):
                    nodes = np.flatnonzero(dom[lv] == d)
                    t = trial(nodes, p, e)
                    if t is not None:
                        trials.append(((sum(c for c, _, _ in t[0]), d), t[0], nodes, t[1]))
                if trials:
                    _, res, nodes, f = min(trials, key=lambda t: t[0])
                    F[nodes] = f
                    break
        if res is None and gd[p] != REQ:
            t = trial(np.arange(len(F)), p, e)
            if t is not None:
                res, F = t
        if res is not None:
            out[p:e] = res
    return out, F


def ref_domain_plan(topo, free, hold, mem, domain, pods, lvl, gang, gd, W, base=0):
    """kgpu_preempt_plan_gang_domain, ranked on tuples.  A member is ref_preempt of that pod alone over the allowed nodes
    under (F, H), then the update rule: its victims' GPUs are free, the GPUs S taken, neither evictable again; a run is
    all or nothing.  A member gives (L, |V|, cost, node id, S) and its victims; a constrained gang's trial in domain d
    scores (L_d, V_d, C_d, d): the largest L and the sums of |V| and cost.  The smallest trial wins; with none, REQUIRED
    leaves the gang out and PREFERRED plans it over every node.  Returns ([((cost, node id, S), victims) or None], F,
    H)."""
    F = np.array(free, np.int32)
    H = np.full((len(F), 8), -1, np.int32) if hold is None else np.array(hold, np.int32)
    out = [None] * len(pods)

    def run(nodes, p, e):
        f, h, res = F.copy(), H.copy(), []
        for q in range(p, e):
            keys, vic = ref_preempt(topo[nodes], f[nodes], pods[q:q + 1], lvl[q:q + 1], h[nodes], W,
                                    mem=None if mem is None else mem[nodes])
            if keys[0] == NO_FIT:
                return None
            [(cost, i, S)] = as_tuples(keys)
            n, v = int(nodes[i]), int(vic[0])
            R = [g for g in range(8) if not (f[n] >> g) & 1 and h[n, g] >= 0 and (v >> (h[n, g] & 7)) & 1]
            L = max((int(h[n, g]) >> 3 for g in R), default=0)
            f[n] = (int(f[n]) | sum(1 << g for g in R)) & ~S & 0xFF
            h[n, [g for g in range(8) if (S >> g) & 1 or g in R]] = -1
            res.append(((L, bin(v).count("1"), cost, base + n, S), v))
        return res, f, h

    domains = sorted(set(int(d) for d in domain) - {-1})
    for p, e in all_runs(gang):
        res = None
        if gd[p] != 0:
            trials = []
            for d in domains:
                t = run(np.flatnonzero(np.asarray(domain) == d), p, e)
                if t is not None:
                    m = [x for x, _ in t[0]]
                    trials.append(((max(x[0] for x in m), sum(x[1] for x in m), sum(x[2] for x in m), d), t))
            if trials:
                res = min(trials, key=lambda t: t[0])[1]
        if res is None and gd[p] != REQ:
            res = run(np.arange(len(F)), p, e)
        if res is not None:
            out[p:e] = [(x[2:], v) for x, v in res[0]]
            F, H = res[1], res[2]
    return out, F, H


# ---- the edge node in a domain --------------------------------------------------------------------------------------------
def with_edge_domain(topo, free, mem, dom, pods, gang, gd, extra=()):
    """The cluster with edge_matrix()'s node (all 8 GPUs free, EDGE_MEM MiB per GPU) inserted at node EDGE, in the
    domains (every level) of the first node with a level-0 domain, and a REQUIRED gang of one k = 8 member that needs
    EDGE_NEED MiB put first: only the edge node holds it, so under WIDE its cost needs 17 bits.  Without mem every other
    GPU gets the tiny clusters' largest memory, which leaves their pods as they were.  extra: per-pod arrays (gang_level,
    lvl) that get a 0 / 1 for the new pod, returned after the rest."""
    N = len(free)
    mem = np.full((N, 8), 81_920, np.int32) if mem is None else mem
    dom = np.asarray(dom, np.int32)
    two = dom.ndim == 2
    d2 = np.atleast_2d(dom)
    src = int(np.flatnonzero(d2[0] >= 0)[0])
    d2 = np.insert(d2, EDGE, d2[:, src], axis=1)
    topo = np.insert(np.asarray(topo, np.int32), EDGE, edge_matrix(), axis=0)
    free = np.insert(np.asarray(free, np.int32), EDGE, 0xFF)
    mem = np.insert(mem, EDGE, EDGE_MEM, axis=0)
    pods = np.concatenate([synth.make_pods(np.array([8], np.int32)), pods]).astype(np.int32)
    pods[0, 3] = EDGE_NEED
    pods[:, 1] = np.arange(len(pods))
    gang = np.concatenate([[int(gang.max()) + 1], gang]).astype(np.int32)
    gd = np.concatenate([[REQ], gd]).astype(np.int32)
    extra = tuple(np.concatenate([[v], np.asarray(a)]).astype(np.int32) for a, v in extra)
    return (topo, free, mem, d2 if two else d2[0], pods, gang, gd) + extra


def check_edge(name, keys, topo, free, base):
    """The edge gang took the edge node, and the table does what it is there for (check_reached)."""
    assert keys[0] != NO_FIT and (int(keys[0]) >> 8 & 0xFFFFFFFF) == base + EDGE and int(keys[0]) & 0xFF == 0xFF
    if name in WIDE:
        assert int(keys[0]) >> 40 >= 1 << 16 and int(keys[0]) >> 40 == 28 * int(W_of(name)[9])
    check_reached(name, keys, topo, free)


# ---- CPU: the references under every table ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_place_references(place_twin, name):
    W = W_of(name)
    for seed in range(8):
        topo, free, mem, dom, pods, gang, gd = with_edge_domain(*GD.tiny_cluster(seed))
        base = top_base(len(free))
        want, wf = GD.brute_force(topo, free, pods, gang, gd, dom, mem=mem, base=base, W=W)
        keys, f = place_twin(topo, free, pods, gang, gd, dom, mem=mem, base=base, W=W)
        assert (keys == want).all() and (f == wf).all(), seed
        ref, rf = ref_domain_place(topo, free, pods, gang, gd, dom, W, mem=mem, base=base)
        assert as_tuples(want) == ref and (wf == rf).all(), seed
        check_edge(name, want, topo, free, base)


@pytest.mark.parametrize("name", NAMES)
def test_levels_references(levels_twin, name):
    W = W_of(name)
    for seed in range(9):
        topo, free, mem, dom, pods, gang, gd, gl = GL.tiny_cluster(seed)
        topo, free, mem, dom, pods, gang, gd, gl = with_edge_domain(topo, free, mem, dom, pods, gang, gd, extra=((gl, 0),))
        base = top_base(len(free))
        want, wf = GL.brute_force_levels(topo, free, pods, gang, gd, gl, dom, mem=mem, base=base, W=W)
        keys, f = levels_twin(topo, free, pods, gang, gd, gl, dom, mem=mem, base=base, W=W)
        assert (keys == want).all() and (f == wf).all(), seed
        ref, rf = ref_domain_place(topo, free, pods, gang, gd, dom, W, gl=gl, mem=mem, base=base)
        assert as_tuples(want) == ref and (wf == rf).all(), seed
        check_edge(name, want, topo, free, base)


@pytest.mark.parametrize("name", NAMES)
def test_plan_references(plans, name):
    W = W_of(name)
    domain_plan, _, snapshot = plans
    for seed in range(10):
        topo, free, hold, mem, dom, pods, lvl, gang, gd = PD.tiny_cluster(seed)
        topo, free, mem, dom, pods, gang, gd, lvl = with_edge_domain(topo, free, mem, dom, pods, gang, gd, extra=((lvl, 1),))
        hold = np.insert(hold, EDGE, -1, axis=0)
        base = top_base(len(free))
        c = (topo, free, hold, mem, dom, pods, lvl, gang, gd)
        want = PD.brute_force(snapshot, *c, base=base, W=W)
        got = domain_plan(*c, base=base, W=W)
        for g, w in zip(got, want):
            assert (g == w).all(), seed
        ref, rf, rh = ref_domain_plan(*c, W, base=base)
        assert [None if k == NO_FIT else (t, int(v)) for k, t, v in zip(want[0], as_tuples(want[0]), want[1])] == ref, seed
        assert (want[2] == rf).all() and (want[3] == rh).all(), seed
        check_edge(name, want[0], topo, free, base)


# ---- CPU: the emulated kernels on the named cases ------------------------------------------------------------------------------
# The hand-made cases of the three files take well under a second each in the emulator: they run under every table, at
# node_id_base 0 and at the top of the 32-bit range.  The generated ones (hundreds of nodes, up to 1100 pods) take seconds
# each, and each file already runs them under the default table at two low bases: here each runs once, at the top base,
# under the table (and, for levels, the walk) named beside it, so that together they cover every table and both walks.
LARGE_PLACE = {"views": "mixed", "chunk": "zero", "interleaved": "flat_max"}
LARGE_LEVELS = {"large_domain": ("general_edge", False), "chunk": ("zero", True), "levels1": ("random2", True),
                "levels2": ("byte_edge", True), "levels3_mem": ("one_level", False), "levels4": ("mixed", True),
                "levels4_mem": ("flat_max", False)}
LARGE_PLAN = {"views": "one_level", "chunk": "flat_max", "interleaved": "random1"}


def emulated_params(cases, large):
    """(table, case, large) for every table on the hand-made cases, then the generated cases with their own table."""
    small = [(name, case, False) for name in NAMES for case in sorted(set(cases) - set(large))]
    big = [((t if isinstance(t, str) else t[0]), case, True) for case, t in sorted(large.items())]
    return small + big


def test_large_cases_cover_every_table():
    for cases, large in ((GD.EMU_CASES, LARGE_PLACE), (GL.EMU_CASES, LARGE_LEVELS), (PD.EMU_CASES, LARGE_PLAN)):
        assert set(large) < set(cases)
    names = set(LARGE_PLACE.values()) | set(LARGE_PLAN.values()) | {t for t, _ in LARGE_LEVELS.values()}
    # the default table: test_gang_domain, test_gang_domain_levels and test_preempt_plan_domain
    assert names == set(NAMES) - {"default"} and {f for _, f in LARGE_LEVELS.values()} == {False, True}
    assert "large_domain" in LARGE_LEVELS and not LARGE_LEVELS["large_domain"][1]       # spines of 512: chunked by size


@pytest.mark.parametrize("name, case, large", emulated_params(GD.EMU_CASES, LARGE_PLACE))
def test_emulated_place(place_emu, place_twin, name, case, large):
    W = W_of(name)
    topo, free, mem, domain, pods, gang, gd = GD.EMU_CASES[case]()
    for base in (top_base(len(free)),) if large else (0, top_base(len(free))):
        keys, f, _ = GD.emu_place(place_emu, topo, free, pods, gang, gd, domain, mem=mem, base=base, W=W)
        want, wf = place_twin(topo, free, pods, gang, gd, domain, mem=mem, base=base, W=W)
        assert (keys == want).all() and (f == wf).all(), base


@pytest.mark.parametrize("name, case, large", emulated_params(GL.EMU_CASES, LARGE_LEVELS))
def test_emulated_levels(levels_emu, levels_twin, name, case, large):
    """Each level's walk picked by its largest domain, and the chunked walk forced on every level."""
    W = W_of(name)
    topo, free, mem, dom, pods, gang, gd, gl = GL.EMU_CASES[case]()
    top = top_base(len(free))
    runs = ((top, LARGE_LEVELS[case][1]),) if large else ((0, False), (0, True), (top, False), (top, True))
    for base, forced in runs:
        keys, f, _ = GL.emu_place(levels_emu, topo, free, pods, gang, gd, gl, dom, mem=mem, base=base, force_chunked=forced, W=W)
        want, wf = levels_twin(topo, free, pods, gang, gd, gl, dom, mem=mem, base=base, W=W)
        assert (keys == want).all() and (f == wf).all(), (base, forced)


@pytest.mark.parametrize("name, case, large", emulated_params(PD.EMU_CASES, LARGE_PLAN))
def test_emulated_plan(plan_emu, plans, name, case, large):
    W = W_of(name)
    c = PD.EMU_CASES[case]()
    for base in (top_base(len(c[1])),) if large else (0, top_base(len(c[1]))):
        keys, vic, F, H, _ = PD.emu_plan(plan_emu, *c, base=base, W=W)
        want = plans[0](*c, base=base, W=W)
        assert (keys == want[0]).all() and (vic == want[1]).all() and (F == want[2]).all() and (H == want[3]).all(), base


# ---- CPU: the domain id decides a tie ------------------------------------------------------------------------------------------
def tie_cluster():
    """Four racks of four nodes whose ids fall as the node indices rise (rack 3 holds nodes 0-3), in two spines (spine 0:
    racks 0 and 1).  A gang of five k = 8 members that only a spine holds, then constrained gangs of k = 1..4 that
    several racks hold, and a pod on its own in between."""
    topo, _, _ = synth.gen_c2(N=16, P=0, seed=5)
    free = np.full(16, 0xFF, np.int32)
    free[12:16] = [0x5A, 0xF0, 0xFF, 0x81]                  # rack 0: the lowest node and the lowest mask are not the first
    dom = np.array([3 - np.arange(16) // 4, 1 - np.arange(16) // 8], np.int32)
    ks = [8, 8, 8, 8, 8,  2, 3, 1,  4, 4,  2,  1, 1, 1, 1,  4, 2, 4]
    gang = [4, 4, 4, 4, 4, 1, 1, 1, 2, 2, 0, 3, 3, 3, 3, 5, 5, 5]
    gd = [PREF] * 5 + [REQ] * 3 + [PREF] * 2 + [0] + [REQ] * 4 + [REQ] * 3
    gl = [1] * 5 + [0] * 3 + [1] * 2 + [0] + [0] * 4 + [1] * 3
    return topo, free, dom, synth.make_pods(np.array(ks, np.int32)), np.array(gang, np.int32), np.array(gd, np.int32), \
        np.array(gl, np.int32)


def tie_expect(free, dom, pods, gang, gd, gl, base):
    """The zero table's answer: a member takes the lowest node with k free GPUs and on it the lowest k of them; a
    constrained gang takes the lowest level, then the lowest domain id, where every member finds one.  Returns (keys,
    masks after, per constrained gang the number of domains that fit it on the level it took)."""
    F = [int(f) for f in free]
    keys = [NO_FIT] * len(pods)
    fits = []

    def place(nodes, p, e):
        f, out = list(F), []
        for k in pods[p:e, 0].tolist():
            n = next((n for n in nodes if 0 <= k <= bin(f[n]).count("1")), None)
            if n is None:
                return None
            S = sum(sorted(1 << i for i in range(8) if (f[n] >> i) & 1)[:k])
            f[n] &= ~S
            out.append(np.uint64((base + n) << 8 | S))
        return out, f

    for p, e in all_runs(gang):
        res = None
        if gd[p] != 0:
            for lv in range(int(gl[p]) + 1):
                ok = {d: r for d in sorted(set(dom[lv].tolist()) - {-1})
                      if (r := place(np.flatnonzero(dom[lv] == d).tolist(), p, e)) is not None}
                if ok:
                    res = ok[min(ok)]
                    fits.append(len(ok))
                    break
        if res is None and gd[p] != REQ:
            res = place(range(len(F)), p, e)
        if res is not None:
            keys[p:e], F = res
    return np.array(keys, np.uint64), np.array(F, np.int32), fits


def test_zero_table_tie_goes_to_the_lowest_domain_id(place_emu, place_twin, levels_emu, levels_twin, plans, plan_emu):
    """Placement (level 0, and climbing to the spines), and plans with nothing to evict: the twins and the emulated
    kernels give tie_expect's keys, at node ids near the top of the range."""
    W = W_of("zero")
    topo, free, dom, pods, gang, gd, gl = tie_cluster()
    base = top_base(len(free))
    want, wf, fits = tie_expect(free, dom[:1], pods, gang, gd, gl * 0, base)
    assert len(fits) == 4 and min(fits) >= 2 and (want != NO_FIT).all()
    got = [place_twin(topo, free, pods, gang, gd, dom[0], base=base, W=W),
           GD.emu_place(place_emu, topo, free, pods, gang, gd, dom[0], base=base, W=W)[:2],
           GD.brute_force(topo, free, pods, gang, gd, dom[0], base=base, W=W)]
    lvl = np.full(len(pods), 2, np.int32)
    for plan in (plans[0](topo, free, None, None, dom[0], pods, lvl, gang, gd, base=base, W=W),
                 PD.emu_plan(plan_emu, topo, free, None, None, dom[0], pods, lvl, gang, gd, base=base, W=W)):
        assert (plan[1] == 0).all()
        got.append((plan[0], plan[2]))
    for k, f in got:
        assert (k == want).all() and (f == wf).all()
    want, wf, fits = tie_expect(free, dom, pods, gang, gd, gl, base)
    assert len(fits) == 5 and min(fits) >= 2 and (want != NO_FIT).all()
    lv = GL.outcome_levels(want - np.uint64(base << 8), gang, gd, dom)
    assert lv == [1, 0, 0, 0, 0]                            # the 8-GPU gang fits no rack, both spines
    for forced in (False, True):
        k, f, _ = GL.emu_place(levels_emu, topo, free, pods, gang, gd, gl, dom, base=base, force_chunked=forced, W=W)
        assert (k == want).all() and (f == wf).all()
    k, f = levels_twin(topo, free, pods, gang, gd, gl, dom, base=base, W=W)
    assert (k == want).all() and (f == wf).all()


def test_zero_table_plan_tie_with_evictions(plans, plan_emu):
    """Every node is held whole by one level-1 owner; level-2 members evict.  Three racks of three nodes, ids falling as
    the node indices rise: trials of equal (L_d, V_d) tie on cost 0, so the lowest rack id that fits wins, and in it each
    member takes the lowest node with the smallest (L, |V|), then the lowest mask."""
    W = W_of("zero")
    topo, _, _ = synth.gen_c2(N=9, P=0, seed=6)
    free = np.zeros(9, np.int32)
    hold = np.full((9, 8), 1 << 3, np.int32)
    dom = (2 - np.arange(9) // 3).astype(np.int32)
    pods = synth.make_pods(np.array([8, 4, 4, 8, 8, 2, 2], np.int32))
    lvl = np.full(7, 2, np.int32)
    gang = np.array([1, 1, 1, 2, 2, 3, 3], np.int32)
    gd = np.array([REQ] * 5 + [PREF] * 2, np.int32)
    base = top_base(9)
    # gang 1 in rack 0 (nodes 6-8): evicts node 6, evicts node 7 for 0x0F, takes 7's other half without evicting;
    # gang 2 fits rack 0 no more (node 8 alone): rack 1, nodes 3 and 4; gang 3: rack 0 again, on node 8
    want = [(6, 0xFF, 1), (7, 0x0F, 1), (7, 0xF0, 0), (3, 0xFF, 1), (4, 0xFF, 1), (8, 0x03, 1), (8, 0x0C, 0)]
    c = (topo, free, hold, None, dom, pods, lvl, gang, gd)
    for got in (plans[0](*c, base=base, W=W), PD.emu_plan(plan_emu, *c, base=base, W=W)):
        assert [(int(k) >> 8 & 0xFFFFFFFF, int(k) & 0xFF, int(v)) for k, v in zip(got[0], got[1])] == \
            [(base + n, S, v) for n, S, v in want]
        assert (got[0] >> np.uint64(40) == 0).all()
    ref, _, _ = ref_domain_plan(*c, W, base=base)
    assert [(t[1] - base, t[2], v) for t, v in ref] == want


# ---- the summed gang cost past 2^31 ---------------------------------------------------------------------------------------------
CD_J = 18_731                                               # members, and nodes per domain
CD_EDGE = 28 * 4095                                         # a k = 8 member's cost on an edge node under one_level


def cd_cluster():
    """Two domains of CD_J nodes, all 8 GPUs free.  Domain 0 (nodes 0 .. j - 1): every node edge_matrix(), so
    C_0 = j * 114 660 > 2^31.  Domain 1: the same but for its last two nodes, whose pairs sit at level 12 (weight 0 under
    one_level), so C_1 = (j - 2) * 114 660 < 2^31.  One REQUIRED gang of j k = 8 members."""
    j = CD_J
    topo = np.tile(edge_matrix(), (2 * j, 1)).astype(np.int32)
    topo[2 * j - 2:] = edge_matrix(12)
    dom = (np.arange(2 * j) >= j).astype(np.int32)
    pods = synth.make_pods(np.full(j, 8, np.int32))
    return topo, np.full(2 * j, 0xFF, np.int32), dom, pods, np.ones(j, np.int32), np.full(j, REQ, np.int32)


def cd_expect():
    """The keys of the gang in domain 1: the two free-of-cost nodes first, then the edge nodes in order."""
    j = CD_J
    C0, C1 = j * CD_EDGE, (j - 2) * CD_EDGE
    assert C0 == 2_147_696_460 > 2**31 > C1 == 2_147_467_140
    assert C0 - 2**32 < 0 < C1 and C0 % 2**31 < C1                # a signed or a 31-bit sum would pick domain 0
    nodes = [2 * j - 2, 2 * j - 1] + list(range(j, 2 * j - 2))
    costs = [0, 0] + [CD_EDGE] * (j - 2)
    keys = np.array([c << 40 | n << 8 | 0xFF for c, n in zip(costs, nodes)], np.uint64)
    assert sum(costs) == C1
    return keys, np.where(np.arange(2 * j) < j, 0xFF, 0).astype(np.int32)


def test_summed_cost_past_2_31_twins(place_twin, plans):
    W = W_of("one_level")
    topo, free, dom, pods, gang, gd = cd_cluster()
    want, wf = cd_expect()
    keys, f = place_twin(topo, free, pods, gang, gd, dom, W=W)
    assert (keys == want).all() and (f == wf).all()
    hold = np.full((len(free), 8), 1 << 3, np.int32)           # one level-1 owner (owner 0) holds every node
    keys, vic, F, H = plans[0](topo, np.zeros(len(free), np.int32), hold, None, dom, pods, np.full(len(pods), 2, np.int32), gang, gd, W=W)
    assert (keys == want).all() and (vic == 1).all() and (F == 0).all()
    assert (H[:CD_J] == hold[:CD_J]).all() and (H[CD_J:] == -1).all()           # every member evicted its node's owner


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
def gang_modes(gang, seed, levels=1):
    rng = np.random.default_rng(seed)
    gd, gl = np.zeros(len(gang), np.int32), np.zeros(len(gang), np.int32)
    for a, e in GD.runs(gang):
        gd[a:e] = rng.integers(0, 3)
        gl[a:e] = rng.integers(0, levels) if gd[a] else 0
    return gd, gl


def place_cluster(use_mem, N=20_000, P=3000, seed=3):
    """gen_gangs with racks of 32 inside spines of 1024 (gen_domain_levels; the spines take the chunked walk); with
    use_mem, C6's GPU memory and min_mem, and the edge node and its gang (with_edge_domain)."""
    topo, free, pods, gang = synth.gen_gangs(N=N, P=P)
    mem = None
    if use_mem:
        _, _, mem, c6 = synth.gen_c6(N=N, P=P)
        pods[:, 3] = c6[:, 3]
    gd, gl = gang_modes(gang, seed, levels=2)
    dom = synth.gen_domain_levels(N, (32, 1024))
    if use_mem:
        topo, free, mem, dom, pods, gang, gd, gl = with_edge_domain(topo, free, mem, dom, pods, gang, gd, extra=((gl, 0),))
    return topo, free, mem, dom, pods, gang, gd, gl


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_place_against_twins(place_twin, levels_twin, name):
    """kgpu_place_batch_gang_domain and kgpu_place_batch_gang_levels, dry run (masks unchanged) and committed, bit-exact
    against the twins; the spine level's chunk-minimum launches are counted."""
    from kubegpu_b200.scorer import Scorer
    W = W_of(name)
    for use_mem in (False, True):
        topo, free, mem, dom, pods, gang, gd, gl = place_cluster(use_mem)
        for base in (0, top_base(len(free))):
            one, one_f = place_twin(topo, free, pods, gang, gd, dom[0], mem=mem, base=base, W=W)
            two, two_f = levels_twin(topo, free, pods, gang, gd, gl, dom, mem=mem, base=base, W=W)
            check_reached(name, two, topo if use_mem else None, free)
            if use_mem:
                check_edge(name, one, topo, free, base)
            with Scorer((0,)) as s:
                s.set_weights(W)
                s.upload_nodes(topo, free, node_id_base=base)
                if mem is not None:
                    s.upload_gpu_memory(mem)
                s.upload_domains(dom)
                n0 = s.kernel_launches
                assert (s.place_batch(pods, gang=gang, gang_domain=gd, dry_run=True) == one).all()
                n1 = s.kernel_launches
                assert (s.get_free_masks() == free).all()
                assert (s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=gl, dry_run=True) == two).all()
                n2 = s.kernel_launches
                assert (s.get_free_masks() == free).all()
                # each gang bound to level 1 adds that level's trial and one domain_chunk_min launch (spines > 256 nodes)
                climbing = sum(1 for a, _ in GD.runs(gang) if gl[a] == 1)
                assert climbing > 10 and (n2 - n1) - (n1 - n0) == 2 * climbing
                assert (s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=gl) == two).all()
                assert (s.get_free_masks() == two_f).all()
                s.set_free_masks(np.arange(len(free)), free)
                assert (s.place_batch(pods, gang=gang, gang_domain=gd) == one).all()
                assert (s.get_free_masks() == one_f).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_plan_against_twin(plans, name):
    W = W_of(name)
    N = 20_000
    for use_mem, base in ((False, top_base(N)), (True, 0), (True, top_base(N))):
        topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs(N=N, P=3000)
        mem = None
        if use_mem:
            mem = synth.gen_gpu_memory(N)
            pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[synth.rand_below(synth.SEED_C6, 14, len(pods), 7)]
        gd, _ = gang_modes(gang, 7)
        dom = synth.gen_domains(N, 32)
        want_k, want_v, _, _ = plans[0](topo, free, hold, mem, dom, pods, lvl, gang, gd, base=base, W=W)
        check_reached(name, want_k[want_v != 0])
        with PD._scorer(topo, free, hold, mem, dom, base=base) as s:
            s.set_weights(W)
            keys, vic = s.preempt_plan(pods, lvl, gang=gang, gang_domain=gd)
            assert (keys == want_k).all() and (vic == want_v).all(), (use_mem, base)
            assert (s.get_free_masks() == free).all()


@pytest.mark.gpu
def test_gpu_weight_changes_on_a_live_handle(place_twin, levels_twin, plans):
    """One upload of nodes, holders and a two-level domain table, then table after table in LIVE_ORDER with mask updates
    before and after each change: the three domain calls equal their twins under the new table each time.  Every other
    step commits the level placement, so the handle's masks move on."""
    from kubegpu_b200.scorer import Scorer
    N = 8000
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs(N=N, P=1500)
    dom = synth.gen_domain_levels(N, (16, 512))
    gd, gl = gang_modes(gang, 9, levels=2)
    rng = np.random.default_rng(10)
    fm = free.copy()
    base = top_base(N)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, fm, node_id_base=base)
        s.upload_holders(hold)
        s.upload_domains(dom)
        for step, name in enumerate(LIVE_ORDER):
            W = W_of(name)
            s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=gl, dry_run=True)     # under the previous table
            upd = rng.choice(N, size=8, replace=False)
            fm[upd] = rng.integers(0, 256, size=8)
            s.set_free_masks(upd, fm[upd])
            s.set_weights(W)
            upd = rng.choice(N, size=8, replace=False)
            fm[upd] = rng.integers(0, 256, size=8)
            s.set_free_masks(upd, fm[upd])
            want, _ = place_twin(topo, fm, pods, gang, gd, dom[0], base=base, W=W)
            assert (s.place_batch(pods, gang=gang, gang_domain=gd, dry_run=True) == want).all(), name
            pk, pv, _, _ = plans[0](topo, fm, hold, None, dom[0], pods, lvl, gang, gd, base=base, W=W)
            keys, vic = s.preempt_plan(pods, lvl, gang=gang, gang_domain=gd)
            assert (keys == pk).all() and (vic == pv).all(), name
            want, wf = levels_twin(topo, fm, pods, gang, gd, gl, dom, base=base, W=W)
            assert (s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=gl, dry_run=step % 2 == 0) == want).all(), name
            if step % 2:
                fm = wf
            assert (s.get_free_masks() == fm).all(), name


@pytest.mark.gpu
def test_gpu_summed_cost_past_2_31_place():
    from kubegpu_b200.scorer import Scorer
    topo, free, dom, pods, gang, gd = cd_cluster()
    want, wf = cd_expect()
    with Scorer((0,)) as s:
        s.set_weights(W_of("one_level"))
        s.upload_nodes(topo, free)
        s.upload_domains(dom)
        t0 = time.perf_counter()
        keys = s.place_batch(pods, gang=gang, gang_domain=gd)
        print("kgpu_place_batch_gang_domain, %d members: %.1f s" % (CD_J, time.perf_counter() - t0))
        assert (keys == want).all() and (s.get_free_masks() == wf).all()


@pytest.mark.gpu
def test_gpu_summed_cost_past_2_31_plan():
    topo, free, dom, pods, gang, gd = cd_cluster()
    want, wf = cd_expect()
    hold = np.full((len(free), 8), 1 << 3, np.int32)
    with PD._scorer(topo, np.zeros(len(free), np.int32), hold, None, dom) as s:
        s.set_weights(W_of("one_level"))
        t0 = time.perf_counter()
        keys, vic = s.preempt_plan(pods, np.full(len(pods), 2, np.int32), gang=gang, gang_domain=gd)
        print("kgpu_preempt_plan_gang_domain, %d members: %.1f s" % (CD_J, time.perf_counter() - t0))
        assert (keys == want).all() and (vic == 1).all()
