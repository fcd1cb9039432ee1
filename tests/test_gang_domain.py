"""Gangs inside one network domain (kgpu_place_batch_gang_domain): a constrained gang takes the domain whose trial
placement costs least, or, with none, NO_FIT (REQUIRED) or the plain gang placement (PREFERRED).  CPU: the twin
(tests/gang_domain_twin/gang_domain_twin.c, built with the oracle) against a Python brute force of the definition and
against its consequences P2-P5, and the emulated launch plan (tests/gang_domain_emu) against the twin.  GPU: the device path
bit-exact against the twin at C2 and C3 size, P1-P5, dry runs, rejected inputs, the domain table's lifetime, and the
host mirror."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import cpu_libs
import gang_domain_libs
from kubegpu_b200 import _lib, synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLI = os.path.join(ROOT, "kubegpu_b200", "lib", "kgpu_sched_cli")
NO_FIT = np.uint64(0xFFFFFFFFFFFFFFFF)
REQ, PREF = 1, 2


def _p(a, t=ctypes.c_int32):
    return None if a is None else a.ctypes.data_as(ctypes.POINTER(t))


def _i32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.int32)


def _W(W=None):
    """The link-weight table W as int32[16]; None is the default table."""
    from oracle import oracle_b
    return np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS if W is None else W, dtype=np.int32)


@pytest.fixture(scope="session")
def twin():
    """place(topo, free, pods, gang, gd, domain, mem=None, base=0, W=None) -> (keys, free_after)."""
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
    """kgpu_place_batch_gang's twin (tests/gang_twin): the plain gang result."""
    L = cpu_libs.twin("gang")

    def place(topo, free, pods, gang, mem=None, base=0, W=None):
        topo, pods, gang, mem = (_i32(a) for a in (topo, pods, gang, mem))
        f = np.array(free, dtype=np.int32, copy=True)
        keys = np.empty(len(pods), dtype=np.uint64)
        L.gang_twin_place_batch(_p(topo), _p(f), _p(mem), len(f), base, _p(pods), _p(gang), len(pods), _p(_W(W)), _p(keys, ctypes.c_uint64))
        return keys, f
    return place


def runs(gang):
    """[(first, end)] of the nonzero gang runs."""
    out, p = [], 0
    while p < len(gang):
        e = p + 1
        while e < len(gang) and gang[e] == gang[p]:
            e += 1
        if gang[p] != 0:
            out.append((p, e))
        p = e
    return out


def node_of(key, base=0):
    return int((int(key) >> 8) & 0xFFFFFFFF) - base


def random_batch(P, seed, share=0.6):
    """Gang ids (runs of 1..6 pods, ids 1, 2, ...) and gang_domain values (0, 1 or 2 per gang, 0 for solo pods)."""
    rng = np.random.default_rng(seed)
    gang, gd = np.zeros(P, np.int32), np.zeros(P, np.int32)
    p, gid = 0, 0
    while p < P:
        n = int(rng.integers(1, 7))
        if rng.random() < share:
            gid += 1
            gang[p:p + n] = gid
            gd[p:p + n] = int(rng.integers(0, 3))
        p += n
    return gang, gd


# ---- a Python brute force of the definition ------------------------------------------------------------------------------
def brute_force(topo, free, pods, gang, gd, domain, mem=None, base=0, W=None):
    from oracle import oracle_b
    W = _W(W)
    F = [int(x) for x in free]
    N = len(F)
    keys = np.full(len(pods), NO_FIT, dtype=np.uint64)

    def nkey(n, mask, k, need):
        if mem is not None and need > 0:
            mask &= sum(1 << i for i in range(8) if mem[n][i] >= need)
        return oracle_b.node_key(topo[n], mask, k, W)

    def place(members, state, nodes):
        """members in order on a copy of state over `nodes`: (keys, state, cost), or None if one misses."""
        st, out, cost = list(state), [], 0
        for q in members:
            k, need = int(pods[q, 0]), int(pods[q, 3])
            if not 0 <= k <= 8:
                return None
            best = int(NO_FIT)
            for n in nodes:
                nk = nkey(n, st[n], k, need)
                if nk != 0xFFFFFFFF:
                    best = min(best, ((nk >> 8) << 40) | ((base + n) << 8) | (nk & 0xFF))
            if best == int(NO_FIT):
                return None
            out.append(best)
            cost += best >> 40
            n = node_of(best, base)
            st[n] = (st[n] & 0xFF) & ~(best & 0xFF)
        return out, st, cost

    domains = sorted(set(int(d) for d in domain) - {-1})
    p = 0
    while p < len(pods):
        e = p + 1
        while gang[p] != 0 and e < len(pods) and gang[e] == gang[p]:
            e += 1
        res = None
        if gd[p] != 0:
            trials = []
            for d in domains:
                r = place(range(p, e), F, [n for n in range(N) if domain[n] == d])
                if r is not None:
                    trials.append((r[2], d, r))
            if trials:
                res = min(trials, key=lambda t: (t[0], t[1]))[2]
        if res is None and (gd[p] != REQ):
            res = place(range(p, e), F, range(N))
        if res is not None:
            keys[p:e], F = res[0], res[1]
        p = e
    return keys, np.array(F, dtype=np.int32)


def tiny_cluster(seed, N=10):
    rng = np.random.default_rng(seed)
    topo, _, _ = synth.gen_c2(N=N, P=0, seed=1000 + seed)
    free = rng.integers(0, 256, N).astype(np.int32)
    free[rng.random(N) < 0.3] = 0xFF
    domain = rng.integers(-1, 3, N).astype(np.int32)
    ks = rng.choice([0, 1, 2, 2, 4, 4, 8, 9], 14).astype(np.int32)
    pods = synth.make_pods(ks)
    mem = None
    if seed % 2:
        mem = rng.choice([16_384, 32_768, 81_920], (N, 8)).astype(np.int32)
        pods[:, 3] = rng.choice([0, 0, 20_000, 40_000], len(ks))
    gang, gd = random_batch(len(ks), seed, share=0.8)
    return topo, free, mem, domain, pods, gang, gd


@pytest.mark.parametrize("seed", range(8))
def test_twin_equals_brute_force(twin, seed):
    topo, free, mem, domain, pods, gang, gd = tiny_cluster(seed)
    want, wf = brute_force(topo, free, pods, gang, gd, domain, mem=mem, base=5)
    keys, f = twin(topo, free, pods, gang, gd, domain, mem=mem, base=5)
    assert (keys == want).all() and (f == wf).all()


# ---- the consequences of the definition, on the twin -----------------------------------------------------------------------
def c2_batch(N=400, P=300, seed=11, size=8):
    topo, free, pods = synth.gen_c2(N=N, P=P, seed=synth.SEED_C2 + seed)
    pods[:, 0] = np.where(pods[:, 0] == 1, 2, pods[:, 0])
    gang, gd = random_batch(P, seed)
    return topo, free, pods, gang, gd, synth.gen_domains(N, size, seed=seed)


def test_twin_p2_one_domain_is_plain_gangs(twin, gang_twin):
    topo, free, pods, gang, gd, _ = c2_batch()
    want, wf = gang_twin(topo, free, pods, gang)
    for mode in (REQ, PREF):
        keys, f = twin(topo, free, pods, gang, np.where(gang != 0, mode, 0), np.zeros(len(free), np.int32))
        assert (keys == want).all() and (f == wf).all()


def test_twin_p3_p4_required_gangs_sit_in_one_domain(twin):
    topo, free, pods, gang, _, domain = c2_batch()
    domain[::7] = -1
    gd = np.where(gang != 0, REQ, 0).astype(np.int32)
    for dom in (domain, np.arange(len(free), dtype=np.int32)):
        keys, _ = twin(topo, free, pods, gang, gd, dom)
        placed = 0
        for a, e in runs(gang):
            if (keys[a:e] == NO_FIT).all():
                continue
            placed += 1
            doms = {int(dom[node_of(k)]) for k in keys[a:e]}
            assert len(doms) == 1 and -1 not in doms
        assert placed > 10


def test_twin_p5_preferred_is_required_or_plain(twin, gang_twin):
    """Gang by gang on the running state: PREFERRED gives the REQUIRED result when that places the gang, the plain gang
    result otherwise."""
    topo, free, pods, gang, _, domain = c2_batch(P=200)
    state = free.copy()
    fell_back = kept = 0
    for a, e in runs(gang):
        sl = slice(a, e)
        g = gang[sl]
        rk, rf = twin(topo, state, pods[sl], g, np.full(e - a, REQ, np.int32), domain)
        pk, pf = twin(topo, state, pods[sl], g, np.full(e - a, PREF, np.int32), domain)
        if (rk != NO_FIT).all():
            assert (pk == rk).all() and (pf == rf).all()
            kept += 1
        else:
            gk, gf = gang_twin(topo, state, pods[sl], g)
            assert (pk == gk).all() and (pf == gf).all()
            fell_back += (gk != NO_FIT).all()
        state = pf
    assert kept > 5 and fell_back > 0


def test_gen_domains_deals_nodes_into_scattered_domains():
    dom = synth.gen_domains(1000, 32)
    assert dom.dtype == np.int32 and dom.min() == 0 and dom.max() == 31
    counts = np.bincount(dom)
    assert (counts[:-1] == 32).all() and counts[-1] == 1000 - 31 * 32
    assert not all(np.ptp(np.flatnonzero(dom == d)) < 32 for d in range(31))
    assert (synth.gen_domains(1000, 32) == dom).all() and not (synth.gen_domains(1000, 32, seed=1) == dom).all()


# ---- the launch plan on the CPU (tests/gang_domain_emu) --------------------------------------------------------------------------------
def _uniform(N, shape=((4, 4),)):
    return np.stack([synth.shape_matrix([list(g) for g in shape])] * N)


def case_required_one_domain():
    topo, _, _ = synth.gen_c2(N=16, P=0)
    free = np.full(16, 0x0F, np.int32)
    free[8:12] = 0xFF                       # only domain 2 holds an 8-GPU member
    pods = synth.make_pods(np.array([8, 4, 4, 2], np.int32))
    gang, gd = np.array([1, 1, 1, 0], np.int32), np.array([REQ, REQ, REQ, 0], np.int32)
    return topo, free, None, np.arange(16, dtype=np.int32) // 4, pods, gang, gd


def case_required_nowhere():
    topo, _, _ = synth.gen_c2(N=16, P=0)
    pods = synth.make_pods(np.array([1] + [8] * 5 + [2], np.int32))
    gang = np.array([0] + [3] * 5 + [0], np.int32)
    return topo, np.full(16, 0xFF, np.int32), None, np.arange(16, dtype=np.int32) // 4, pods, gang, np.where(gang != 0, REQ, 0)


def case_preferred_fallback_fits():
    t = case_required_nowhere()
    return t[:6] + (np.where(t[5] != 0, PREF, 0),)


def case_preferred_fallback_fails():
    topo, _, _ = synth.gen_c2(N=16, P=0)
    pods = synth.make_pods(np.array([2] + [8] * 17 + [4], np.int32))
    gang = np.array([0] + [4] * 17 + [0], np.int32)
    return topo, np.full(16, 0xFF, np.int32), None, np.arange(16, dtype=np.int32) // 4, pods, gang, np.where(gang != 0, PREF, 0)


def case_tie():
    """Two identical domains: the lower id wins although its nodes have the higher ids."""
    topo = _uniform(8)
    domain = np.array([1, 1, 1, 1, 0, 0, 0, 0], np.int32)
    pods = synth.make_pods(np.array([4, 4, 2], np.int32))
    return topo, np.full(8, 0xFF, np.int32), None, domain, pods, np.array([1, 1, 1], np.int32), np.full(3, REQ, np.int32)


def case_k0_k9():
    topo, _, _ = synth.gen_c2(N=12, P=0)
    free = np.full(12, 0xFF, np.int32)
    free[:4] = 0
    domain = np.array([0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3], np.int32)
    ks = [0, 4, 0, 2,  4, 9, 1,  9, 4,  0, 8]
    gang = [1, 1, 1, 1, 2, 2, 2, 3, 3, 4, 4]
    gd = [REQ] * 4 + [REQ] * 3 + [PREF] * 2 + [PREF] * 2
    return topo, free, None, domain, synth.make_pods(np.array(ks, np.int32)), np.array(gang, np.int32), np.array(gd, np.int32)


def case_two_members_one_node():
    topo = _uniform(8, ((8,),))
    free = np.array([0x0F, 0x0F, 0xFF, 0x3F, 0xFF, 0xFF, 0xFF, 0xFF], np.int32)
    pods = synth.make_pods(np.array([2, 2, 2, 4], np.int32))
    domain = np.array([0, 0, 1, 1, 2, 2, 3, 3], np.int32)
    return topo, free, None, domain, pods, np.ones(4, np.int32), np.full(4, REQ, np.int32)


def case_scattered_tiles():
    """A domain whose nodes sit in three tiles, the cheaper nodes of the cluster in none."""
    N = 128 * 3 + 5
    topo, free, _ = synth.gen_c2(N=N, P=0)
    free[:] = 0x0F
    domain = np.full(N, -1, np.int32)
    domain[[3, 200, 300, N - 1]] = 0
    domain[[5, 6, 7]] = 1
    free[[3, 200, 300, N - 1]] = 0xFF
    pods = synth.make_pods(np.array([8, 8, 4, 8, 2, 4], np.int32))
    gang = np.array([1, 1, 1, 1, 0, 2], np.int32)
    gd = np.array([REQ, REQ, REQ, REQ, 0, PREF], np.int32)
    return topo, free, None, domain, pods, gang, gd


def case_minus_one_nodes():
    topo, _, _ = synth.gen_c2(N=20, P=0)
    free = np.full(20, 0x33, np.int32)
    domain = np.array([-1] * 10 + [0] * 5 + [1] * 5, np.int32)
    free[:10] = 0xFF                        # the best nodes belong to no domain
    pods = synth.make_pods(np.array([2, 2, 2, 4, 4, 8, 2], np.int32))
    gang = np.array([1, 1, 1, 2, 2, 0, 3], np.int32)
    gd = np.array([REQ, REQ, REQ, REQ, REQ, 0, PREF], np.int32)
    return topo, free, None, domain, pods, gang, gd


def case_views():
    topo, free, mem, pods = synth.gen_c6(N=300, P=160)
    pods[:, 3] = np.array([0, 8_000, 20_000, 40_000])[np.arange(160) % 4]
    gang, gd = random_batch(160, 9)
    return topo, free, mem, synth.gen_domains(300, 16), pods, gang, gd


def case_chunk():
    """A constrained gang across pod 1024, between plain gangs and solo pods."""
    topo, free, pods = synth.gen_c2(N=256, P=1040)
    gang = np.zeros(1040, np.int32)
    gd = np.zeros(1040, np.int32)
    pods[::3, 0] = -1
    gang[1000:1010] = 1
    gang[1018:1027], gd[1018:1027] = 2, REQ
    gang[1027:1031], gd[1027:1031] = 3, PREF
    gang[1031:1034] = 4
    return topo, free, None, synth.gen_domains(256, 16), pods, gang, gd


def case_interleaved():
    topo, free, pods = synth.gen_c2(N=500, P=240, seed=synth.SEED_C2 + 7)
    gang, gd = random_batch(240, 4)
    return topo, free, None, synth.gen_domains(500, 8, seed=4), pods, gang, gd


EMU_CASES = {
    "required_one_domain": case_required_one_domain,
    "required_nowhere": case_required_nowhere,
    "preferred_fallback_fits": case_preferred_fallback_fits,
    "preferred_fallback_fails": case_preferred_fallback_fails,
    "tie": case_tie,
    "k0_k9": case_k0_k9,
    "two_members_one_node": case_two_members_one_node,
    "scattered_tiles": case_scattered_tiles,
    "minus_one_nodes": case_minus_one_nodes,
    "views": case_views,
    "chunk": case_chunk,
    "interleaved": case_interleaved,
}


@pytest.fixture(scope="module")
def emu():
    return gang_domain_libs.emu()


def emu_place(emu, topo, free, pods, gang, gd, domain, mem=None, base=0, W=None):
    topo, pods, gang, gd, domain, mem = (_i32(a) for a in (topo, pods, gang, gd, domain, mem))
    f = np.array(free, dtype=np.int32, copy=True)
    keys = np.empty(len(pods), dtype=np.uint64)
    steps = emu.emu_place_batch_gang_domain(_p(topo), _p(f), _p(mem), len(f), base, _p(domain), _p(pods), _p(gang), _p(gd), len(pods),
                                            _p(_W(W)), _p(keys, ctypes.c_uint64))
    assert steps >= 0
    return keys, f, steps


@pytest.mark.parametrize("base", [0, 21])
@pytest.mark.parametrize("name", sorted(EMU_CASES))
def test_emulated_plan_matches_twin(emu, twin, name, base):
    topo, free, mem, domain, pods, gang, gd = EMU_CASES[name]()
    keys, f, steps = emu_place(emu, topo, free, pods, gang, gd, domain, mem=mem, base=base)
    want, wf = twin(topo, free, pods, gang, gd, domain, mem=mem, base=base)
    assert (keys == want).all() and (f == wf).all()
    assert steps == sum(1 for a, _ in runs(gang) if gd[a] != 0) > 0


def test_emulated_cases_are_what_they_claim(twin):
    """Each hand-made case, as the twin places it."""
    def go(case):
        topo, free, mem, domain, pods, gang, gd = case()
        keys, f = twin(topo, free, pods, gang, gd, domain, mem=mem)
        return keys, f, free, domain
    k, _, _, dom = go(case_required_one_domain)
    assert {int(dom[node_of(x)]) for x in k[:3]} == {2}
    k, f, free, _ = go(case_required_nowhere)
    assert (k[1:6] == NO_FIT).all() and k[0] != NO_FIT and k[6] != NO_FIT
    k, f, _, dom = go(case_preferred_fallback_fits)
    assert (k[1:6] != NO_FIT).all() and len({int(dom[node_of(x)]) for x in k[1:6]}) > 1
    k, f, _, _ = go(case_preferred_fallback_fails)
    assert (k[1:18] == NO_FIT).all() and k[18] != NO_FIT
    k, _, _, _ = go(case_tie)
    assert {node_of(x) for x in k} <= {4, 5, 6, 7}
    k, _, _, dom = go(case_k0_k9)
    d = int(dom[node_of(k[1])])                     # k = 0: cost 0, no GPUs, the lowest node of the gang's domain
    assert node_of(k[0]) == node_of(k[2]) == int(np.flatnonzero(dom == d)[0]) and int(k[0]) >> 40 == 0 and k[0] & 0xFF == 0
    assert (k[4:9] == NO_FIT).all() and (k[9:] != NO_FIT).all()
    k, _, _, _ = go(case_two_members_one_node)
    assert len({node_of(x) for x in k[:3]}) < 3
    k, _, _, dom = go(case_scattered_tiles)
    assert {node_of(x) // 128 for x in k[:4]} >= {0, 1, 2} and {int(dom[node_of(x)]) for x in k[:4]} == {0}
    k, _, _, dom = go(case_minus_one_nodes)
    assert -1 not in {int(dom[node_of(x)]) for x in k[:5]} and dom[node_of(k[5])] == -1


def test_emulated_dry_run_then_commit(emu, twin):
    """A dry run places on a copy of the masks (as libkgpu does): the committing run then places the same keys."""
    topo, free, mem, domain, pods, gang, gd = case_interleaved()
    dry, df, _ = emu_place(emu, topo, free.copy(), pods, gang, gd, domain)
    keys, f, _ = emu_place(emu, topo, free, pods, gang, gd, domain)
    assert (dry == keys).all() and (df == f).all()


@pytest.mark.parametrize("seed", range(3))
def test_emulated_random_batches(emu, twin, seed):
    rng = np.random.default_rng(seed)
    N, P = int(rng.integers(50, 400)), int(rng.integers(20, 200))
    topo, free, mem, pods = synth.gen_c6(N=N, P=P, seed=synth.SEED_C6 + seed)
    if seed == 0:
        mem, pods[:, 3] = None, 0
    gang, gd = random_batch(P, seed + 100)
    domain = synth.gen_domains(N, int(rng.choice([1, 4, 8, 32])), seed=seed)
    domain[rng.random(N) < 0.1] = -1
    keys, f, _ = emu_place(emu, topo, free, pods, gang, gd, domain, mem=mem, base=seed)
    want, wf = twin(topo, free, pods, gang, gd, domain, mem=mem, base=seed)
    assert (keys == want).all() and (f == wf).all()


# ---- build products --------------------------------------------------------------------------------------------------------
def test_domain_kernels_have_no_local_memory():
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or libkgpu.so missing")
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    lines, found = out.splitlines(), set()
    for i, line in enumerate(lines):
        m = re.search(r"Function _ZN4kgpu\d+(domain_trial|domain_commit)\S*:", line)
        if m:
            found.add(m.group(1))
            assert re.search(r"STACK:0\b", lines[i + 1]) and re.search(r"LOCAL:0\b", lines[i + 1]), lines[i + 1]
    assert found == {"domain_trial", "domain_commit"}


# ---- the device path ---------------------------------------------------------------------------------------------------------
def c2_full(use_mem, seed=5):
    topo, free, pods, gang = synth.gen_gangs()
    mem = None
    if use_mem:
        _, _, mem, c6 = synth.gen_c6(N=len(free), P=len(pods))
        pods[:, 3] = c6[:, 3]
    gd = np.zeros(len(pods), np.int32)
    mode = np.random.default_rng(seed).integers(0, 3, len(pods))
    for a, e in runs(gang):
        gd[a:e] = mode[a]
    return topo, free, mem, pods, gang, gd, synth.gen_domains(len(free), 32)


@pytest.mark.gpu
@pytest.mark.parametrize("use_mem", [False, True])
def test_c2_size_against_twin(twin, use_mem):
    from kubegpu_b200.scorer import Scorer
    topo, free, mem, pods, gang, gd, domain = c2_full(use_mem)
    want, wf = twin(topo, free, pods, gang, gd, domain, mem=mem)
    kinds = [(gd[a], bool((want[a:e] != NO_FIT).all())) for a, e in runs(gang)]
    assert (REQ, True) in kinds and (REQ, False) in kinds and (PREF, True) in kinds
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        if mem is not None:
            s.upload_gpu_memory(mem)
        s.upload_domains(domain)
        dry = s.place_batch(pods, gang=gang, gang_domain=gd, dry_run=True)
        assert (dry == want).all() and (s.get_free_masks() == free).all()
        got = s.place_batch(pods, gang=gang, gang_domain=gd)
        assert (got == want).all() and (s.get_free_masks() == wf).all()


@pytest.mark.gpu
def test_c3_size_against_twin(twin):
    from kubegpu_b200.scorer import Scorer
    topo, free, pods = synth.gen_c3(N=1_000_000, P=1500)
    gang, gd = random_batch(len(pods), 3)
    domain = synth.gen_domains(len(free), 32)
    want, wf = twin(topo, free, pods, gang, gd, domain)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_domains(domain)
        assert (s.place_batch(pods, gang=gang, gang_domain=gd) == want).all() and (s.get_free_masks() == wf).all()


@pytest.mark.gpu
def test_p1_no_constraint_is_place_batch_gang():
    from kubegpu_b200.scorer import Scorer
    topo, free, pods, gang = synth.gen_gangs(N=20_000, P=3000)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_domains(synth.gen_domains(len(free), 32))
        s.place_batch(pods, gang=gang, dry_run=True)
        n0 = s.kernel_launches
        want = s.place_batch(pods, gang=gang, dry_run=True)
        per_call = s.kernel_launches - n0
        for gd in (None, np.zeros(len(pods), np.int32)):
            n1 = s.kernel_launches
            got = s.place_batch(pods, gang=gang, gang_domain=gd, dry_run=True)
            assert (got == want).all() and s.kernel_launches - n1 == per_call
        s.place_batch(pods, gang=gang, gang_domain=np.zeros(len(pods), np.int32))
        wf = s.get_free_masks()
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.place_batch(pods, gang=gang)
        assert (s.get_free_masks() == wf).all()


@pytest.mark.gpu
def test_p2_to_p5_on_the_device(twin, gang_twin):
    from kubegpu_b200.scorer import Scorer
    topo, free, pods, gang, _, domain = c2_batch(N=3000, P=1500, size=16)
    domain[::9] = -1
    N = len(free)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        plain = s.place_batch(pods, gang=gang, dry_run=True)
        s.upload_domains(np.zeros(N, np.int32))
        for mode in (REQ, PREF):                                    # P2
            assert (s.place_batch(pods, gang=gang, gang_domain=np.where(gang != 0, mode, 0), dry_run=True) == plain).all()
        req = np.where(gang != 0, REQ, 0).astype(np.int32)
        for dom in (domain, np.arange(N, dtype=np.int32)):          # P3, P4
            s.upload_domains(dom)
            keys = s.place_batch(pods, gang=gang, gang_domain=req, dry_run=True)
            for a, e in runs(gang):
                if (keys[a:e] != NO_FIT).all():
                    doms = {int(dom[node_of(k)]) for k in keys[a:e]}
                    assert len(doms) == 1 and -1 not in doms
        s.upload_domains(domain)                                     # P5, one gang per call on the running state
        for a, e in runs(gang)[:40]:
            g = np.full(e - a, 1, np.int32)
            r = s.place_batch(pods[a:e], gang=g, gang_domain=np.full(e - a, REQ, np.int32), dry_run=True)
            want = r if (r != NO_FIT).all() else s.place_batch(pods[a:e], gang=g, dry_run=True)
            assert (s.place_batch(pods[a:e], gang=g, gang_domain=np.full(e - a, PREF, np.int32)) == want).all()


@pytest.mark.gpu
def test_rejected_inputs():
    from kubegpu_b200.scorer import KgpuError, Scorer
    topo, free, pods = synth.gen_c2(N=1000, P=6)
    gang = np.array([1, 1, 0, 2, 2, 2], np.int32)
    bad = [
        ([1, 1, 0, 3, 3, 3], "is not 0, REQUIRED (1) or PREFERRED (2)"),
        ([-1, -1, 0, 0, 0, 0], "is not 0, REQUIRED (1) or PREFERRED (2)"),
        ([1, 1, 2, 0, 0, 0], "on a pod without a gang"),
        ([1, 2, 0, 0, 0, 0], "disagree on gang_domain"),
    ]
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        for gd, msg in bad:
            with pytest.raises(KgpuError) as e:
                s.place_batch(pods, gang=gang, gang_domain=np.array(gd, np.int32))
            assert e.value.code == _lib.ERR_INVALID and msg in str(e.value), str(e.value)
        with pytest.raises(KgpuError) as e:
            s.place_batch(pods, gang_domain=np.array([1, 0, 0, 0, 0, 0], np.int32))
        assert "on a pod without a gang" in str(e.value)
        with pytest.raises(KgpuError) as e:
            s.place_batch(pods, gang=np.array([3, 3, 0, 4, 3, 3], np.int32), gang_domain=np.zeros(6, np.int32))
        assert "two separate runs" in str(e.value)
        big = synth.make_pods(np.zeros(37_001, np.int32))
        with pytest.raises(KgpuError) as e:
            s.place_batch(big, gang=np.ones(37_001, np.int32), gang_domain=np.ones(37_001, np.int32))
        assert "more than 37000" in str(e.value)
        many7 = synth.make_pods(np.ones(8, np.int32))
        many7[:, 3] = np.arange(1, 9) * 1000
        with pytest.raises(KgpuError) as e:
            s.place_batch(many7, gang=np.ones(8, np.int32), gang_domain=np.ones(8, np.int32))
        assert "distinct min_mem" in str(e.value)
        for dom, msg in (([5] * 999 + [1000], "domain[999] = 1000"), ([-2] + [0] * 999, "domain[0] = -2")):
            with pytest.raises(KgpuError) as e:
                s.upload_domains(np.array(dom, np.int32))
            assert e.value.code == _lib.ERR_INVALID and msg in str(e.value), str(e.value)
        with pytest.raises(ValueError):
            s.upload_domains(np.zeros(999, np.int32))
        assert (s.get_free_masks() == free).all()


@pytest.mark.gpu
def test_domain_table_lifetime():
    """A bad upload leaves the table as it was; kgpu_upload_nodes resets it to all -1; mask changes leave it alone."""
    from kubegpu_b200.scorer import KgpuError, Scorer
    topo = _uniform(8)
    free = np.full(8, 0xFF, np.int32)
    pods = synth.make_pods(np.array([4, 4], np.int32))
    g, req = np.ones(2, np.int32), np.full(2, REQ, np.int32)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        assert (s.place_batch(pods, gang=g, gang_domain=req, dry_run=True) == NO_FIT).all()      # no domains yet
        s.upload_domains(np.array([-1, -1, -1, -1, 3, 3, 3, 3], np.int32))
        with pytest.raises(KgpuError):
            s.upload_domains(np.array([0] * 7 + [8], np.int32))
        s.set_free_masks(np.arange(4), np.full(4, 0xFF, np.int32))
        keys = s.place_batch(pods, gang=g, gang_domain=req, dry_run=True)
        assert {node_of(k) for k in keys} <= {4, 5, 6, 7}
        s.upload_nodes(topo, free)
        assert (s.place_batch(pods, gang=g, gang_domain=req, dry_run=True) == NO_FIT).all()
        assert (s.place_batch(pods, gang=g, gang_domain=np.full(2, PREF, np.int32), dry_run=True) != NO_FIT).all()


@pytest.mark.gpu
def test_two_device_handle_is_refused():
    import torch
    from kubegpu_b200.scorer import KgpuError, Scorer
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    topo, free, pods = synth.gen_c2(N=100, P=2)
    with Scorer((0, 1)) as s:
        s.upload_nodes(topo, free)
        for call in (lambda: s.upload_domains(np.zeros(100, np.int32)),
                     lambda: s.place_batch(pods, gang=np.ones(2, np.int32), gang_domain=np.ones(2, np.int32))):
            with pytest.raises(KgpuError) as e:
                call()
            assert e.value.code == _lib.ERR_STATE


@pytest.mark.gpu
def test_host_mirror_places_gangs_in_domains(twin, oracle_b):
    """sched_cli: `domain NODE NAME` and `gangdomain=`: names map to ids in sorted order, members move up to their gang's
    first member with their gang domain, ProposeBatch proposes what PlaceBatch places, and bad requests are errors."""
    from test_gang_placement import _node_line
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-s", "-C", ROOT, "kubegpu_b200/lib/kgpu_sched_cli"])
    ids = ["GPU-%02d" % i for i in range(8)]
    shapes = {"A": [[2, 2], [2, 2]], "B": [[4], [2, 2]], "C": [[4], [4]], "D": [[8]]}
    doms = {"A": "rack-b", "B": "rack-a", "C": "rack-a"}            # D in none; ids: rack-a 0, rack-b 1
    spec = [("s1", 2, 0, None), ("g1a", 4, 7, "required"), ("s2", 1, 0, None), ("g1b", 4, 7, "required"),
            ("g2a", 4, 9, "preferred"), ("g2b", 4, 9, "preferred"), ("g3a", 8, 11, "required"), ("g3b", 8, 11, "required")]
    names = " ".join(n for n, _, _, _ in spec)
    script = [_node_line(n, sh, ids) for n, sh in shapes.items()]
    script += ["domain %s %s" % kv for kv in doms.items()] + ["domain D"]
    script += ["pod %s gang=%d%s run c req=%d" % (n, g, "" if d is None else " gangdomain=" + d, k) for n, k, g, d in spec]
    script += ["proposebatch " + names, "placebatch " + names,
               "pod bad1 gangdomain=required run c req=1", "placebatch bad1",
               "pod bad2 gang=5 gangdomain=required run c req=1", "pod bad3 gang=5 gangdomain=preferred run c req=1",
               "placebatch bad2 bad3"]
    got = subprocess.run([CLI], input="\n".join(script) + "\n", capture_output=True, text=True, check=True).stdout
    dev = [0, 1, 3, 2, 4, 5, 6, 7]                                  # s1, g1a, g1b, s2, g2a, g2b, g3a, g3b
    pods = synth.make_pods(np.array([spec[i][1] for i in dev], np.int32))
    gang = np.array([[0, 1, 1, 0, 2, 2, 3, 3][j] for j in range(8)], np.int32)
    gd = np.array([0, REQ, REQ, 0, PREF, PREF, REQ, REQ], np.int32)
    topo = np.stack([synth.shape_matrix(sh) for sh in shapes.values()])
    want, _ = twin(topo, np.full(4, 0xFF, np.int32), pods, gang, gd, np.array([1, 0, 0, -1], np.int32))
    by_name = {spec[i][0]: want[j] for j, i in enumerate(dev)}
    assert by_name["g1a"] != NO_FIT and by_name["g2a"] != NO_FIT and by_name["g3a"] == NO_FIT
    lines = []
    for n, _, _, _ in spec:
        u = oracle_b.unpack_key(by_name[n])
        lines.append("  %s fits=0 cost=0 node= mask=0x00" % n if u is None else
                     "  %s fits=1 cost=%d node=%s mask=0x%02x" % (n, u[0], "ABCD"[u[1]], u[2]))
    for cmd in ("proposebatch", "placebatch"):
        out = got.split("> %s %s\n" % (cmd, names))[1].splitlines()
        assert out[0] == "  err=" and out[1:9] == lines, (cmd, out)
    assert "gpu/gpu-gang-domain without gpu/gpu-gang-id" in got.split("> placebatch bad1\n")[1].splitlines()[0]
    assert "disagree on gpu/gpu-gang-domain" in got.split("> placebatch bad2 bad3\n")[1].splitlines()[0]
