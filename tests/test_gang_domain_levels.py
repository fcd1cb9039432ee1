"""Nested network domains (kgpu_upload_domain_levels, kgpu_place_batch_gang_levels): a constrained gang climbs the levels
0..gang_level and takes the cheapest domain of the first level where one fits.  CPU: the twin
(tests/gang_domain_levels_twin/levels_twin.c, which includes the one-level twin) against a Python brute force built on
test_gang_domain.brute_force and against the consequences Q1 and Q3-Q6 of include/kgpu.h; the emulated kernels and launch
plan (tests/gang_domain_levels_emu) against the twin; the table builder's nesting and range checks; synth's nested
domains.  GPU: the device path bit-exact against the twin at C2 and C3 size and on one 20k-node domain, Q1-Q5, level-0
preemption plans, rejected inputs, the table's lifetime, a two-device handle."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import _lib, synth
from test_gang_domain import REQ, PREF, NO_FIT, _W, _i32, _p, brute_force, node_of, random_batch, runs

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_i32p, _u64p, _i64p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int64)
_i64, _int = ctypes.c_int64, ctypes.c_int
# topo, free, mem, n, base, domain, levels, pods, gang, gang_domain, gang_level, P, W, keys
_PLACE = [_i32p, _i32p, _i32p, _i64, _i64, _i32p, _int, _i32p, _i32p, _i32p, _i32p, _i64, _i32p, _u64p]


# ---- the CPU libraries ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def twin():
    """place(topo, free, pods, gang, gd, gl, domain[L, N], mem=None, base=0, W=None) -> (keys, free_after)."""
    L = cpu_libs.twin("gang_domain_levels")
    L.levels_twin_place_batch.restype, L.levels_twin_place_batch.argtypes = None, _PLACE
    return lambda *a, **kw: _run(L.levels_twin_place_batch, *a, **kw)[:2]


@pytest.fixture(scope="session")
def one_level_twin():
    """kgpu_place_batch_gang_domain's twin: place(topo, free, pods, gang, gd, domain[N], mem=None, base=0, W=None) ->
    (keys, free_after)."""
    import gang_domain_libs
    L = gang_domain_libs.twin()

    def place(topo, free, pods, gang, gd, domain, mem=None, base=0, W=None):
        topo, pods, gang, gd, domain, mem = (_i32(a) for a in (topo, pods, gang, gd, domain, mem))
        f = np.array(free, dtype=np.int32, copy=True)
        keys = np.empty(len(pods), dtype=np.uint64)
        L.gang_domain_twin_place_batch(_p(topo), _p(f), _p(mem), len(f), base, _p(domain), _p(pods), _p(gang), _p(gd), len(pods),
                                       _p(_W(W)), _p(keys, ctypes.c_uint64))
        return keys, f
    return place


@pytest.fixture(scope="session")
def gang_twin():
    L = cpu_libs.twin("gang")

    def place(topo, free, pods, gang, W=None):
        topo, pods, gang = (_i32(a) for a in (topo, pods, gang))
        f = np.array(free, dtype=np.int32, copy=True)
        keys = np.empty(len(pods), dtype=np.uint64)
        L.gang_twin_place_batch(_p(topo), _p(f), None, len(f), 0, _p(pods), _p(gang), len(pods), _p(_W(W)), _p(keys, ctypes.c_uint64))
        return keys, f
    return place


@pytest.fixture(scope="session")
def emu():
    src = os.path.join(HERE, "gang_domain_levels_emu", "emu_levels.cc")
    so = os.path.join(cpu_libs._tmpdir(), "libgang_domain_levels_emu.so")
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-I" + os.path.join(HERE, "emu", "stub"),
                           "-I" + os.path.join(HERE, "emu"), "-I" + os.path.join(ROOT, "kubegpu_b200", "csrc"), "-o", so, src])
    L = ctypes.CDLL(so)
    L.emu_place_batch_gang_levels.restype, L.emu_place_batch_gang_levels.argtypes = _int, _PLACE + [_int]
    L.emu_domain_table.restype = _int
    L.emu_domain_table.argtypes = [_i32p, _int, _i64, _i32p, _i64p, _i64p]
    return L


def _run(fn, topo, free, pods, gang, gd, gl, domain, mem=None, base=0, W=None):
    topo, pods, gang, gd, gl, mem = (_i32(a) for a in (topo, pods, gang, gd, gl, mem))
    dom = None if domain is None else _i32(np.atleast_2d(domain))
    f = np.array(free, dtype=np.int32, copy=True)
    keys = np.empty(len(pods), dtype=np.uint64)
    rc = fn(_p(topo), _p(f), _p(mem), len(f), base, _p(dom), 1 if dom is None else dom.shape[0], _p(pods), _p(gang), _p(gd), _p(gl),
            len(pods), _p(_W(W)), _p(keys, ctypes.c_uint64))
    return keys, f, rc


# ---- a brute force of the climb, on test_gang_domain's brute force of one level ------------------------------------------
def brute_force_levels(topo, free, pods, gang, gd, gl, domain, mem=None, base=0, W=None):
    """Run by run on the running state: a constrained gang is test_gang_domain.brute_force with REQUIRED on level 0, 1,
    ... gang_level until one places it; else NO_FIT (REQUIRED) or brute_force's plain gang (PREFERRED)."""
    F = np.array(free, dtype=np.int32)
    keys = np.full(len(pods), NO_FIT, dtype=np.uint64)
    p = 0
    while p < len(pods):
        e = p + 1
        while gang[p] != 0 and e < len(pods) and gang[e] == gang[p]:
            e += 1
        sl = slice(p, e)
        one = lambda mode, lv: brute_force(topo, F, pods[sl], gang[sl], np.full(e - p, mode, np.int32),
                                           domain[lv] if lv >= 0 else np.full(len(F), -1, np.int32), mem=mem, base=base, W=W)
        res = None
        if gd[p] != 0:
            for lv in range(int(gl[p]) + 1):
                k, f = one(REQ, lv)
                if (k != NO_FIT).all():
                    res = (k, f)
                    break
        if res is None and gd[p] != REQ:
            res = one(0, -1)
        if res is not None:
            keys[sl], F = res
        p = e
    return keys, F


def nested_random(rng, N, levels):
    """Tiny random nested domains [levels, N]: ids of level l are 2 * parent + 0/1, some nodes -1 at the lower levels only."""
    dom = np.empty((levels, N), np.int32)
    dom[-1] = rng.integers(-1, 2, N)
    for lv in range(levels - 2, -1, -1):
        up = dom[lv + 1]
        dom[lv] = np.where(up >= 0, 2 * up + rng.integers(0, 2, N), -1)
        dom[lv][rng.random(N) < 0.2] = -1
    return dom


def tiny_cluster(seed, N=12):
    rng = np.random.default_rng(seed)
    topo, _, _ = synth.gen_c2(N=N, P=0, seed=2000 + seed)
    free = rng.integers(0, 256, N).astype(np.int32)
    free[rng.random(N) < 0.3] = 0xFF
    levels = 1 + seed % 3
    domain = nested_random(rng, N, levels)
    ks = rng.choice([0, 1, 2, 2, 4, 4, 8, 9], 14).astype(np.int32)
    pods = synth.make_pods(ks)
    mem = None
    if seed % 2:
        mem = rng.choice([16_384, 32_768, 81_920], (N, 8)).astype(np.int32)
        pods[:, 3] = rng.choice([0, 0, 20_000, 40_000], len(ks))
    gang, gd = random_batch(len(ks), seed, share=0.8)
    gl = random_levels(rng, gang, gd, levels)
    return topo, free, mem, domain, pods, gang, gd, gl


def random_levels(rng, gang, gd, levels):
    gl = np.zeros(len(gang), np.int32)
    for a, e in runs(gang):
        if gd[a] != 0:
            gl[a:e] = rng.integers(0, levels)
    return gl


@pytest.mark.parametrize("seed", range(9))
def test_twin_equals_brute_force(twin, seed):
    topo, free, mem, domain, pods, gang, gd, gl = tiny_cluster(seed)
    want, wf = brute_force_levels(topo, free, pods, gang, gd, gl, domain, mem=mem, base=3)
    keys, f = twin(topo, free, pods, gang, gd, gl, domain, mem=mem, base=3)
    assert (keys == want).all() and (f == wf).all()


# ---- the consequences, on the twin ------------------------------------------------------------------------------------------
def c2_levels(N=600, P=400, seed=11, sizes=(8, 64)):
    topo, free, pods = synth.gen_c2(N=N, P=P, seed=synth.SEED_C2 + seed)
    pods[:, 0] = np.where(pods[:, 0] == 1, 4, pods[:, 0])
    gang, gd = random_batch(P, seed)
    dom = synth.gen_domain_levels(N, sizes, seed=seed)
    dom[0][np.random.default_rng(seed).random(N) < 0.1] = -1
    return topo, free, pods, gang, gd, dom


def test_twin_q1_level_zero_is_one_domain(twin, one_level_twin):
    topo, free, pods, gang, gd, dom = c2_levels()
    want, wf = one_level_twin(topo, free, pods, gang, gd, dom[0])
    for gl in (None, np.zeros(len(pods), np.int32)):
        keys, f = twin(topo, free, pods, gang, gd, gl, dom)
        assert (keys == want).all() and (f == wf).all()


def test_twin_q3_q6(twin):
    """Q3: level 1 = one domain makes REQUIRED r = 1 the PREFERRED r = 0 result; Q6: a failed REQUIRED gang changes
    nothing (the batch with it equals the batch without it)."""
    topo, free, pods, gang, _, dom = c2_levels()
    dom[1] = 0
    member = (gang != 0).astype(np.int32)
    a = twin(topo, free, pods, gang, member * REQ, member, dom)
    b = twin(topo, free, pods, gang, member * PREF, None, dom)
    assert (a[0] == b[0]).all() and (a[1] == b[1]).all()
    keys, f = twin(topo, free, pods, gang, member * REQ, None, dom)
    failed = [(s, e) for s, e in runs(gang) if (keys[s:e] == NO_FIT).all()]
    assert len(failed) > 3
    keep = np.ones(len(pods), bool)
    for s, e in failed:
        keep[s:e] = False
    k2, f2 = twin(topo, free, pods[keep], gang[keep], (member * REQ)[keep], None, dom)
    assert (k2 == keys[keep]).all() and (f2 == f).all()


def test_twin_q4_q5_gang_by_gang(twin, gang_twin):
    """On the running state, gang by gang, with bound r = 1: a placed REQUIRED gang sits in one domain of some level
    l* <= r and the bound l* - 1 fails there (Q4); PREFERRED is REQUIRED when that fits, the plain gang otherwise (Q5)."""
    topo, free, pods, gang, _, dom = c2_levels(P=300)
    state = free.copy()
    seen = {0: 0, 1: 0, "fallback": 0}
    for a, e in runs(gang):
        sl = slice(a, e)
        g, one = gang[sl], np.ones(e - a, np.int32)
        rk, rf = twin(topo, state, pods[sl], g, one * REQ, one, dom)
        pk, pf = twin(topo, state, pods[sl], g, one * PREF, one, dom)
        if (rk != NO_FIT).all():
            [lstar] = outcome_levels(rk, g, one, dom)
            if lstar == 1:
                assert (twin(topo, state, pods[sl], g, one * REQ, one * 0, dom)[0] == NO_FIT).all()
            seen[lstar] += 1
            assert (pk == rk).all() and (pf == rf).all()
        else:
            assert (rf == state).all()
            gk, gf = gang_twin(topo, state, pods[sl], g)
            assert (pk == gk).all() and (pf == gf).all()
            seen["fallback"] += int((gk != NO_FIT).all())
        state = pf
    assert seen[0] > 5 and seen[1] > 0 and seen["fallback"] > 0, seen


def test_gen_domain_levels_nests():
    for sizes in ((32, 1024), (32, 3125), (4, 16, 64, 256)):
        dom = synth.gen_domain_levels(10_000, sizes, seed=3)
        assert dom.shape == (len(sizes), 10_000) and dom.dtype == np.int32
        assert (dom[0] == synth.gen_domains(10_000, sizes[0], seed=3)).all()
        for lv in range(len(sizes) - 1):
            parents = {}
            for d, u in zip(dom[lv].tolist(), dom[lv + 1].tolist()):
                assert parents.setdefault(d, u) == u
        counts = np.bincount(dom[-1])
        assert abs(int(np.median(counts)) - sizes[-1]) <= sizes[-2]
        assert not all(np.ptp(np.flatnonzero(dom[0] == d)) < sizes[0] for d in range(5))
    with pytest.raises(ValueError):
        synth.gen_domain_levels(100, (32, 16))


# ---- the table builder (launch_plan.h: domain_table) -----------------------------------------------------------------------
def table(emu, dom):
    dom = _i32(np.atleast_2d(dom))
    L, n = dom.shape
    D = np.zeros(L, np.int32)
    sizes, info = np.zeros(2, np.int64), np.zeros(6, np.int64)
    kind = emu.emu_domain_table(_p(dom), L, n, _p(D), _p(sizes, ctypes.c_int64), _p(info, ctypes.c_int64))
    return kind, (D.tolist(), sizes.tolist()) if kind == 0 else info.tolist()


def test_table_builder_accepts_nested_levels(emu):
    dom = [[0, 0, -1, 1, 1, -1], [0, 0, 0, 1, 1, 1], [0, 0, 0, 0, 0, 0]]
    assert table(emu, dom) == (0, ([2, 2, 1], [3 + 3 + 2, 4 + 6 + 6]))
    assert table(emu, [[-1] * 4, [2, 2, -1, 0]]) == (0, ([0, 3], [1 + 4, 3]))     # -1 at level 0, set at level 1
    assert table(emu, synth.gen_domain_levels(5000, (32, 1024, 2048)))[0] == 0


def test_table_builder_refuses(emu):
    # out of range: (level, node, -, id)
    assert table(emu, [[0, 0, 0, 0], [0, 0, 4, 0]]) == (1, [1, 2, -1, 4, 0, 0])
    assert table(emu, [[-2, 0, 0, 0]]) == (1, [0, 0, -1, -2, 0, 0])
    # a level-0 domain without a level-1 domain: (level, node, -, id, -1)
    assert table(emu, [[1, 1, 0, 0], [0, -1, 0, 0]]) == (2, [0, 1, -1, 1, -1, 0])
    # a level-1 domain split over two level-2 domains: (level, node, first node, id, its parent, this parent)
    assert table(emu, [[0, 1, 1, 2], [0, 0, 0, 1], [0, 0, 1, 1]]) == (3, [1, 2, 0, 0, 0, 1])


# ---- the launch plan on the CPU -----------------------------------------------------------------------------------------------
def emu_place(emu, topo, free, pods, gang, gd, gl, domain, mem=None, base=0, force_chunked=False, W=None):
    """force_chunked: every level walked by chunk minima, whatever its domains' size."""
    fn = lambda *a: emu.emu_place_batch_gang_levels(*a, int(force_chunked))
    keys, f, launches = _run(fn, topo, free, pods, gang, gd, gl, domain, mem=mem, base=base, W=W)
    assert launches >= 0
    return keys, f, launches


def case_climb():
    """Racks of 2 that hold no 3-member gang, spines of 4 that do; one gang per mode and bound, a -1 rack node that a
    spine still holds, k = 0 and k = 9 members."""
    topo, free, _ = synth.gen_c2(N=16, P=0)
    free[:] = 0xFF
    dom = np.array([np.arange(16) // 2, np.arange(16) // 4, np.zeros(16)], np.int32)
    dom[0][[5, 9]] = -1
    ks = [8, 8, 8,  8, 8, 8,  8, 8, 8,  8, 8, 8,  0, 4, 0,  4, 9,  2]
    gang = [1, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5, 6, 6, 0]
    gd = [REQ] * 3 + [REQ] * 3 + [PREF] * 3 + [PREF] * 3 + [REQ] * 3 + [REQ] * 2 + [0]
    gl = [0] * 3 + [1] * 3 + [0] * 3 + [2] * 3 + [1] * 3 + [2] * 2 + [0]
    return topo, free, None, dom, synth.make_pods(np.array(ks, np.int32)), np.array(gang, np.int32), np.array(gd, np.int32), \
        np.array(gl, np.int32)


def case_two_members_one_node():
    """Members that share a node of the winning level-1 domain: the trial re-scores the node it changed."""
    topo = np.stack([synth.shape_matrix([[8]])] * 8)
    free = np.array([0x0F, 0x0F, 0x0F, 0x3F, 0x0F, 0x0F, 0x03, 0x03], np.int32)     # no rack holds 14 GPUs
    dom = np.array([[0, 0, 1, 1, 2, 2, 3, 3], [0, 0, 0, 0, 1, 1, 1, 1]], np.int32)
    pods = synth.make_pods(np.array([2, 2, 2, 4, 4], np.int32))
    return topo, free, None, dom, pods, np.ones(5, np.int32), np.full(5, REQ, np.int32), np.ones(5, np.int32)


def case_random(levels, seed, use_mem, P=200, N=700):
    rng = np.random.default_rng(seed)
    if use_mem:
        topo, free, mem, pods = synth.gen_c6(N=N, P=P, seed=synth.SEED_C6 + seed)
        pods[:, 3] = np.array([0, 8_000, 20_000, 40_000])[np.arange(P) % 4]
    else:
        topo, free, pods = synth.gen_c2(N=N, P=P, seed=synth.SEED_C2 + seed)
        mem = None
    pods[:, 0] = np.where(pods[:, 0] == 1, 4, pods[:, 0])
    sizes = (4, 16, 64, 256)[4 - levels:] if levels > 1 else (8,)
    dom = synth.gen_domain_levels(N, sizes, seed=seed)
    for lv in range(levels - 1):                # -1 at level lv takes -1 below it, so the levels still nest
        dom[:lv + 1, rng.random(N) < 0.05] = -1
    gang, gd = random_batch(P, seed + 50)
    return topo, free, mem, dom, pods, gang, gd, random_levels(rng, gang, gd, levels)


def case_chunk():
    """Constrained gangs across pod 1024 (the K3 staging chunk), between plain gangs and solo pods."""
    topo, free, pods = synth.gen_c2(N=256, P=1040)
    gang, gd, gl = (np.zeros(1040, np.int32) for _ in range(3))
    pods[::3, 0] = -1
    gang[1000:1010] = 1
    gang[1018:1027], gd[1018:1027], gl[1018:1027] = 2, REQ, 1
    gang[1027:1031], gd[1027:1031], gl[1027:1031] = 3, PREF, 1
    gang[1031:1034] = 4
    return topo, free, None, synth.gen_domain_levels(256, (8, 64)), pods, gang, gd, gl


def case_large_domain():
    """Racks of 8 inside spines of 512 nodes: the spines are walked by chunk minima without forcing."""
    topo, free, mem, dom, pods, gang, gd, gl = case_random(2, 9, True, P=160, N=1100)
    dom = synth.gen_domain_levels(1100, (8, 512), seed=9)
    return topo, free, mem, dom, pods, gang, gd, np.where(gd != 0, 1, 0).astype(np.int32)


EMU_CASES = {
    "large_domain": case_large_domain,
    "climb": case_climb,
    "two_members_one_node": case_two_members_one_node,
    "chunk": case_chunk,
    "levels1": lambda: case_random(1, 1, False),
    "levels2": lambda: case_random(2, 2, False),
    "levels3_mem": lambda: case_random(3, 3, True),
    "levels4": lambda: case_random(4, 4, False),
    "levels4_mem": lambda: case_random(4, 5, True),
}


@pytest.mark.parametrize("base, walk", [(0, "by size"), (21, "by size"), (21, "chunked")])
@pytest.mark.parametrize("name", sorted(EMU_CASES))
def test_emulated_plan_matches_twin(emu, twin, name, base, walk):
    """Both walks against the twin: each level's walk picked by its largest domain, and the chunked walk forced on every
    level (members that share a chunk make the trial rescan it node by node)."""
    topo, free, mem, dom, pods, gang, gd, gl = EMU_CASES[name]()
    keys, f, launches = emu_place(emu, topo, free, pods, gang, gd, gl, dom, mem=mem, base=base, force_chunked=walk == "chunked")
    want, wf = twin(topo, free, pods, gang, gd, gl, dom, mem=mem, base=base)
    assert (keys == want).all() and (f == wf).all()
    steps = [(a, e) for a, e in runs(gang) if gd[a] != 0]
    assert steps and launches >= 2 + sum(int(gl[a]) + 2 for a, _ in steps)


def test_emulated_cases_are_what_they_claim(twin):
    topo, free, mem, dom, pods, gang, gd, gl = case_climb()
    k, _ = twin(topo, free, pods, gang, gd, gl, dom)
    assert (k[0:3] == NO_FIT).all()                                  # REQUIRED r = 0: no rack holds three 8-GPU pods
    assert len({int(dom[1][node_of(x)]) for x in k[3:6]}) == 1       # r = 1: one spine
    assert (k[6:9] != NO_FIT).all()                                   # PREFERRED r = 0: the plain gang
    assert (k[9:12] != NO_FIT).all() and len({int(dom[1][node_of(x)]) for x in k[9:12]}) == 1
    assert (k[15:17] == NO_FIT).all() and k[12] != NO_FIT and int(k[12]) & 0xFF == 0 and int(k[12]) >> 40 == 0
    rack = int(dom[0][node_of(k[13])])                                  # k = 0: the lowest node of the gang's rack
    assert node_of(k[12]) == node_of(k[14]) == int(np.flatnonzero(dom[0] == rack)[0])
    topo, free, mem, dom, pods, gang, gd, gl = case_two_members_one_node()
    k, _ = twin(topo, free, pods, gang, gd, gl, dom)
    assert (k != NO_FIT).all() and len({node_of(x) for x in k}) < 5 and len({int(dom[0][node_of(x)]) for x in k}) > 1


def test_emulated_level_zero_is_the_one_level_launch_plan(emu):
    """gang_level NULL or all 0 on a 3-level table: the keys, masks and launch count of the 1-level table (Q1, Q2)."""
    topo, free, mem, dom, pods, gang, gd, _ = case_random(3, 8, True)
    want = emu_place(emu, topo, free, pods, gang, gd, None, dom[:1], mem=mem)
    for gl in (None, np.zeros(len(pods), np.int32)):
        got = emu_place(emu, topo, free, pods, gang, gd, gl, dom, mem=mem)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all() and got[2] == want[2]


# ---- the device path ---------------------------------------------------------------------------------------------------------
def c2_full(use_mem, seed=5, sizes=(32, 1024)):
    topo, free, pods, gang = synth.gen_gangs()
    mem = None
    if use_mem:
        _, _, mem, c6 = synth.gen_c6(N=len(free), P=len(pods))
        pods[:, 3] = c6[:, 3]
    rng = np.random.default_rng(seed)
    gd, gl = np.zeros(len(pods), np.int32), np.zeros(len(pods), np.int32)
    for a, e in runs(gang):
        gd[a:e] = rng.integers(0, 3)
        gl[a:e] = rng.integers(0, len(sizes)) if gd[a] else 0
    return topo, free, mem, pods, gang, gd, gl, synth.gen_domain_levels(len(free), sizes)


def outcome_levels(keys, gang, gd, dom):
    """Per placed constrained gang, the lowest level whose one domain holds it (or 'across')."""
    out = []
    for a, e in runs(gang):
        if gd[a] == 0 or (keys[a:e] == NO_FIT).any():
            continue
        lv = [l for l in range(len(dom)) if len({int(dom[l][node_of(k)]) for k in keys[a:e]}) == 1
              and dom[l][node_of(keys[a])] >= 0]
        out.append(lv[0] if lv else "across")
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("use_mem", [False, True])
def test_c2_size_against_twin(twin, use_mem):
    from kubegpu_b200.scorer import Scorer
    topo, free, mem, pods, gang, gd, gl, dom = c2_full(use_mem)
    want, wf = twin(topo, free, pods, gang, gd, gl, dom, mem=mem)
    got_levels = outcome_levels(want, gang, gd, dom)
    assert 0 in got_levels and 1 in got_levels
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        if mem is not None:
            s.upload_gpu_memory(mem)
        s.upload_domains(dom)
        dry = s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=gl, dry_run=True)
        assert (dry == want).all() and (s.get_free_masks() == free).all()
        got = s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=gl)
        assert (got == want).all() and (s.get_free_masks() == wf).all()


@pytest.mark.gpu
def test_c3_size_against_twin(twin):
    from kubegpu_b200.scorer import Scorer
    topo, free, pods = synth.gen_c3(N=1_000_000, P=1500)
    gang, gd = random_batch(len(pods), 3)
    dom = synth.gen_domain_levels(len(free), (32, 1024, 16384))
    gl = random_levels(np.random.default_rng(3), gang, gd, 3)
    want, wf = twin(topo, free, pods, gang, gd, gl, dom)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_domains(dom)
        assert (s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=gl) == want).all() and (s.get_free_masks() == wf).all()


@pytest.mark.gpu
def test_one_large_domain_against_twin(twin):
    """Racks of 32 inside one level-1 domain of all 20k nodes: gangs that fit no rack walk the whole domain."""
    from kubegpu_b200.scorer import Scorer
    topo, free, pods, gang = synth.gen_gangs(N=20_000, P=3000)
    dom = synth.gen_domain_levels(len(free), (32,)).repeat(2, axis=0)
    dom[1] = 0
    member = (gang != 0).astype(np.int32)
    gd = member * np.where(np.arange(len(pods)) % 2, REQ, PREF).astype(np.int32)
    for a, e in runs(gang):
        gd[a:e] = gd[a]
    want, wf = twin(topo, free, pods, gang, gd, member, dom)
    assert 1 in outcome_levels(want, gang, gd, dom)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_domains(dom)
        assert (s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=member) == want).all() and (s.get_free_masks() == wf).all()


@pytest.mark.gpu
def test_q1_q2_level_zero_on_the_device():
    """Q1: gang_level None or all 0 is kgpu_place_batch_gang_domain, with the same launch count; Q2: that call reads
    level 0 of a 3-level table and nothing else."""
    from kubegpu_b200.scorer import Scorer
    topo, free, mem, pods, gang, gd, _, dom = c2_full(True, seed=2, sizes=(8, 64, 512))
    pods, gang, gd = pods[:3000], gang[:3000], gd[:3000]
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_gpu_memory(mem)
        s.upload_domains(dom[0])
        s.place_batch(pods, gang=gang, gang_domain=gd, dry_run=True)
        n0 = s.kernel_launches
        want = s.place_batch(pods, gang=gang, gang_domain=gd, dry_run=True)
        per_call = s.kernel_launches - n0
        s.upload_domains(dom)
        n1 = s.kernel_launches
        assert (s.place_batch(pods, gang=gang, gang_domain=gd, dry_run=True) == want).all()            # Q2
        assert s.kernel_launches - n1 == per_call
        n1 = s.kernel_launches                                                                      # Q1
        assert (s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=np.zeros(len(pods), np.int32), dry_run=True) == want).all()
        assert s.kernel_launches - n1 == per_call
        steps = sum(1 for a, _ in runs(gang) if gd[a] != 0)
        n1 = s.kernel_launches
        s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=np.where(gd != 0, 2, 0), dry_run=True)
        # one trial per level, and one chunk-minimum launch for level 2, whose 512-node domains take the chunked walk
        assert s.kernel_launches - n1 == per_call + 3 * steps


@pytest.mark.gpu
def test_q3_q4_q5_on_the_device():
    from kubegpu_b200.scorer import Scorer
    topo, free, pods, gang, _, dom = c2_levels(N=3000, P=1500, sizes=(16, 256))
    member = (gang != 0).astype(np.int32)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        flat = dom.copy()
        flat[1] = 0
        s.upload_domains(flat)                                                                      # Q3
        a = s.place_batch(pods, gang=gang, gang_domain=member * REQ, gang_level=member, dry_run=True)
        b = s.place_batch(pods, gang=gang, gang_domain=member * PREF, gang_level=member * 0, dry_run=True)
        assert (a == b).all()
        s.upload_domains(dom)                                                                       # Q4
        keys = s.place_batch(pods, gang=gang, gang_domain=member * REQ, gang_level=member, dry_run=True)
        lv = outcome_levels(keys, gang, member, dom)
        assert "across" not in lv and lv.count(0) > 5 and lv.count(1) > 0
        for (a0, e), l in zip([r for r in runs(gang) if (keys[r[0]:r[1]] != NO_FIT).all()], lv):
            assert all(dom[l][node_of(k)] >= 0 for k in keys[a0:e])
        state = s.get_free_masks()                                                                  # Q4 l < l*, Q5, Q6
        for a0, e in runs(gang)[:40]:
            g, one = np.ones(e - a0, np.int32), np.ones(e - a0, np.int32)
            r = s.place_batch(pods[a0:e], gang=g, gang_domain=one * REQ, gang_level=one, dry_run=True)
            if (r != NO_FIT).all() and outcome_levels(r, g, one, dom) == [1]:
                assert (s.place_batch(pods[a0:e], gang=g, gang_domain=one * REQ, gang_level=one * 0, dry_run=True) == NO_FIT).all()
            want = r if (r != NO_FIT).all() else s.place_batch(pods[a0:e], gang=g, dry_run=True)
            if (r == NO_FIT).all():
                s.place_batch(pods[a0:e], gang=g, gang_domain=one * REQ, gang_level=one)
                assert (s.get_free_masks() == state).all()
            assert (s.place_batch(pods[a0:e], gang=g, gang_domain=one * PREF, gang_level=one) == want).all()
            state = s.get_free_masks()


@pytest.mark.gpu
def test_preempt_plan_reads_level_zero():
    from kubegpu_b200.scorer import Scorer
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs(N=5000, P=2500)
    dom = synth.gen_domain_levels(len(free), (8, 128))
    gd = np.zeros(len(pods), np.int32)
    for i, (a, e) in enumerate(runs(gang)):
        gd[a:e] = (REQ, PREF, 0)[i % 3]
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_holders(hold)
        s.upload_domains(dom[0])
        want = s.preempt_plan(pods, lvl, gang=gang, gang_domain=gd)
        s.upload_domains(dom)
        got = s.preempt_plan(pods, lvl, gang=gang, gang_domain=gd)
        assert all((x == y).all() for x, y in zip(got, want))


@pytest.mark.gpu
def test_rejected_inputs():
    from kubegpu_b200.scorer import KgpuError, Scorer
    topo, free, pods = synth.gen_c2(N=1000, P=6)
    gang = np.array([1, 1, 0, 2, 2, 2], np.int32)
    gd = np.array([1, 1, 0, 2, 2, 2], np.int32)
    two = synth.gen_domain_levels(1000, (8, 64))
    bad_levels = [
        ([2, 2, 0, 0, 0, 0], "gang_level[0] = 2 is outside 0..1 (the domain table has 2 levels)"),
        ([-1, -1, 0, 0, 0, 0], "gang_level[0] = -1 is outside 0..1"),
        ([0, 0, 1, 0, 0, 0], "gang_level[2] = 1 on a pod without a domain constraint"),
        ([0, 1, 0, 0, 0, 0], "the members of gang 1 disagree on gang_level"),
    ]
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_domains(two)
        for gl, msg in bad_levels:
            with pytest.raises(KgpuError) as e:
                s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=np.array(gl, np.int32))
            assert e.value.code == _lib.ERR_INVALID and msg in str(e.value), str(e.value)
            assert "kgpu_place_batch_gang_levels" in str(e.value)
        with pytest.raises(KgpuError) as e:                                   # the checks of the one-level call
            s.place_batch(pods, gang=gang, gang_domain=np.array([1, 2, 0, 0, 0, 0], np.int32), gang_level=np.zeros(6, np.int32))
        assert "disagree on gang_domain" in str(e.value)
        with pytest.raises(KgpuError) as e:
            s.place_batch(pods, gang_domain=np.zeros(6, np.int32), gang_level=np.array([0, 0, 0, 1, 0, 0], np.int32))
        assert "on a pod without a domain constraint" in str(e.value)
        for kw in ({}, {"gang": gang}):                                       # gang_level without gang_domain
            with pytest.raises(KgpuError) as e:
                s.place_batch(pods, gang_level=np.array([0, 0, 0, 1, 0, 0], np.int32), **kw)
            assert "gang_level[3] = 1 on a pod without a domain constraint" in str(e.value)
        s.upload_domains(two[0])
        with pytest.raises(KgpuError) as e:
            s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=np.array([1, 1, 0, 0, 0, 0], np.int32))
        assert "outside 0..0 (the domain table has 1 level)" in str(e.value)
        uploads = [
            (np.zeros((5, 1000), np.int32), "levels = 5 is outside 1..4"),
            (np.stack([two[0], np.where(np.arange(1000) == 7, 1000, two[1])]), "domain[1][7] = 1000 is neither -1 nor 0..999"),
            (np.stack([two[0], np.where(np.arange(1000) == 5, -1, two[1])]), "level 0: node 5 is in domain %d but in no level-1" % two[0][5]),
        ]
        split = two.copy()
        i = int(np.flatnonzero(two[0] == two[0][0])[1])
        split[1][i] = (two[1][0] + 1) % (two[1].max() + 1)
        uploads.append((split, "level 0: domain %d is not nested: node 0 is in level-1 domain %d, node %d in %d"
                        % (two[0][0], two[1][0], i, split[1][i])))
        for dom, msg in uploads:
            with pytest.raises(KgpuError) as e:
                s.upload_domains(dom)
            assert e.value.code == _lib.ERR_INVALID and msg in str(e.value), str(e.value)
            assert "kgpu_upload_domain_levels" in str(e.value)
        with pytest.raises(ValueError):
            s.upload_domains(np.zeros((2, 999), np.int32))
        assert (s.get_free_masks() == free).all()


@pytest.mark.gpu
def test_table_lifetime():
    """A refused upload leaves the levels as they were, kgpu_upload_nodes resets to one level of -1, and the one-level
    upload replaces a multi-level table."""
    from kubegpu_b200.scorer import KgpuError, Scorer
    topo = np.stack([synth.shape_matrix([[4, 4]])] * 8)
    free = np.full(8, 0xFF, np.int32)
    pods = synth.make_pods(np.array([8, 8, 8], np.int32))
    g, req = np.ones(3, np.int32), np.full(3, REQ, np.int32)
    dom = np.array([[0, 0, 1, 1, 2, 2, 3, 3], [0, 0, 0, 0, 1, 1, 1, 1]], np.int32)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        with pytest.raises(KgpuError):
            s.place_batch(pods, gang=g, gang_domain=req, gang_level=g)           # one level until an upload
        s.upload_domains(dom)
        with pytest.raises(KgpuError):
            s.upload_domains(np.array([[0] * 8, [0] * 7 + [1]], np.int32))
        s.set_free_masks(np.arange(2), np.zeros(2, np.int32))
        keys = s.place_batch(pods, gang=g, gang_domain=req, gang_level=g, dry_run=True)
        assert (keys != NO_FIT).all() and {node_of(k) for k in keys} <= {4, 5, 6, 7}
        assert (s.place_batch(pods, gang=g, gang_domain=req, gang_level=g * 0, dry_run=True) == NO_FIT).all()
        s.upload_domains(dom[0])
        with pytest.raises(KgpuError):
            s.place_batch(pods, gang=g, gang_domain=req, gang_level=g)
        s.upload_domains(dom)
        s.upload_nodes(topo, free)
        with pytest.raises(KgpuError):
            s.place_batch(pods, gang=g, gang_domain=req, gang_level=g)
        assert (s.place_batch(pods, gang=g, gang_domain=req, gang_level=g * 0, dry_run=True) == NO_FIT).all()


@pytest.mark.gpu
def test_two_device_handle_is_refused():
    import torch
    from kubegpu_b200.scorer import KgpuError, Scorer
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    topo, free, pods = synth.gen_c2(N=100, P=2)
    with Scorer((0, 1)) as s:
        s.upload_nodes(topo, free)
        for call in (lambda: s.upload_domains(np.zeros((2, 100), np.int32)),
                     lambda: s.place_batch(pods, gang=np.ones(2, np.int32), gang_domain=np.ones(2, np.int32),
                                           gang_level=np.zeros(2, np.int32))):
            with pytest.raises(KgpuError) as e:
                call()
            assert e.value.code == _lib.ERR_STATE


@pytest.mark.gpu
def test_host_mirror_places_gangs_in_nested_domains(twin, oracle_b):
    """sched_cli: `domain NODE NAME0 NAME1` and `gangdomainlevel=`: names map to ids per level in sorted order, a
    required gang that no rack holds climbs to the spine, one held to racks finds none, ProposeBatch proposes what PlaceBatch places, and bad requests
    are errors (a level without a gang domain, members that disagree, a level in a preemption plan)."""
    from test_gang_placement import _node_line
    CLI = os.path.join(ROOT, "kubegpu_b200", "lib", "kgpu_sched_cli")
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-s", "-C", ROOT, "kubegpu_b200/lib/kgpu_sched_cli"])
    ids = ["GPU-%02d" % i for i in range(8)]
    shapes = {"A": [[4], [4]], "B": [[8]], "C": [[2, 2], [2, 2]], "D": [[4], [2, 2]]}
    doms = {"A": "rack-b spine", "B": "rack-b spine", "C": "rack-a spine", "D": "- spine"}   # ids: rack-a 0, rack-b 1
    spec = [("g1a", 8, 7, "required", 1), ("g1b", 8, 7, "required", 1), ("g1c", 8, 7, "required", 1),
            ("g2a", 8, 9, "required", 0), ("g2b", 8, 9, "required", 0), ("s1", 2, 0, None, 0)]
    names = " ".join(n for n, _, _, _, _ in spec)
    script = [_node_line(n, sh, ids) for n, sh in shapes.items()]
    script += ["domain %s %s" % kv for kv in doms.items()]
    script += ["pod %s gang=%d%s%s run c req=%d" % (n, g, "" if d is None else " gangdomain=" + d,
                                                    " gangdomainlevel=%d" % r if r else "", k) for n, k, g, d, r in spec]
    script += ["proposebatch " + names, "placebatch " + names,
               "pod bad1 gang=3 gangdomainlevel=1 run c req=1", "placebatch bad1",
               "pod bad2 gang=5 gangdomain=required gangdomainlevel=1 run c req=1",
               "pod bad3 gang=5 gangdomain=required run c req=1", "placebatch bad2 bad3",
               "preemptdomainplan bad2"]
    got = subprocess.run([CLI], input="\n".join(script) + "\n", capture_output=True, text=True, check=True).stdout
    pods = synth.make_pods(np.array([k for _, k, _, _, _ in spec], np.int32))
    gang = np.array([1, 1, 1, 2, 2, 0], np.int32)
    gd = np.array([REQ] * 5 + [0], np.int32)
    gl = np.array([1, 1, 1, 0, 0, 0], np.int32)
    topo = np.stack([synth.shape_matrix(sh) for sh in shapes.values()])
    dom = np.array([[1, 1, 0, -1], [0, 0, 0, 0]], np.int32)
    want, _ = twin(topo, np.full(4, 0xFF, np.int32), pods, gang, gd, gl, dom)
    assert (want[:3] != NO_FIT).all() and (want[3:5] == NO_FIT).all() and want[5] != NO_FIT
    lines = []
    for (n, _, _, _, _), key in zip(spec, want):
        u = oracle_b.unpack_key(key)
        lines.append("  %s fits=0 cost=0 node= mask=0x00" % n if u is None else
                     "  %s fits=1 cost=%d node=%s mask=0x%02x" % (n, u[0], "ABCD"[u[1]], u[2]))
    for cmd in ("proposebatch", "placebatch"):
        out = got.split("> %s %s\n" % (cmd, names))[1].splitlines()
        assert out[0] == "  err=" and out[1:7] == lines, (cmd, out)
    assert "gpu/gpu-gang-domain-level without gpu/gpu-gang-domain" in got.split("> placebatch bad1\n")[1].splitlines()[0]
    assert "disagree on gpu/gpu-gang-domain-level" in got.split("> placebatch bad2 bad3\n")[1].splitlines()[0]
    assert "not supported in preemption plans" in got.split("> preemptdomainplan bad2\n")[1].splitlines()[0]


def test_chunk_min_kernel_has_no_local_memory():
    """domain_chunk_min, the chunked walk's table build (domain_trial and domain_commit are checked by
    test_gang_domain)."""
    import re
    import shutil
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or libkgpu.so missing")
    lines = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout.splitlines()
    found = [i for i, line in enumerate(lines) if re.search(r"Function _ZN4kgpu\d+domain_chunk_min\S*:", line)]
    assert len(found) == 1
    assert re.search(r"STACK:0\b", lines[found[0] + 1]) and re.search(r"LOCAL:0\b", lines[found[0] + 1])
