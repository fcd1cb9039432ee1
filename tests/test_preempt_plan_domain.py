"""Preemption plans for gangs inside one network domain (kgpu_preempt_plan_gang_domain): a constrained gang evicts and
takes its GPUs within the domain whose trial plan scores lowest in (max victim level, victims, cost, domain id), or, with
none, gets NO_FIT (REQUIRED) or the plain gang plan (PREFERRED).  CPU: the twin
(tests/preempt_plan_domain_twin/plan_domain_twin.c) against a Python brute force of the definition built from
single-pod preempt_twin_batch calls, and against the consequences P1-P6; the emulated launch plan
(tests/preempt_plan_domain_emu) against the twin on named cases and random batches; the build products.  GPU: the device
path bit-exact against the twin on gen_preempt_gangs, P1-P5 on the device, rejected inputs, the handle's state, a
two-device handle and the host mirror."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import gang_domain_libs
import preempt_plan_domain_libs
from kubegpu_b200 import _lib, synth
from test_preemption import _row, random_holders

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


def _out(P):
    return np.empty(P, np.uint64), np.empty(P, np.uint32)


def _state(free, hold):
    return np.array(free, np.int32, copy=True), (np.full((len(free), 8), -1, np.int32) if hold is None
                                                 else np.array(hold, np.int32, copy=True))


@pytest.fixture(scope="session")
def plans():
    """(domain_plan, gang_plan, snapshot).  domain_plan(topo, free, hold, mem, domain, pods, lvl, gang, gd, base=0) ->
    (keys, victims, F, H) with the final working state; gang_plan(topo, free, hold, mem, pods, lvl, gang, base=0) ->
    (keys, victims) is preempt_plan_gang_twin; snapshot(topo, free, hold, mem, pods, lvl, base=0) is preempt_twin_batch.
    Each takes W=None, the link-weight table (None: the default)."""
    L = preempt_plan_domain_libs.twin()
    nt = os.cpu_count() or 1

    def domain_plan(topo, free, hold, mem, domain, pods, lvl, gang, gd, base=0, W=None):
        topo, mem, domain, pods, lvl, gang, gd = (_i32(a) for a in (topo, mem, domain, pods, lvl, gang, gd))
        F, H = _state(free, hold)
        keys, vic = _out(len(pods))
        L.preempt_plan_domain_twin(_p(topo), _p(F), _p(mem), _p(H), len(F), base, _p(domain), _p(pods), _p(lvl), _p(gang), _p(gd),
                                   len(pods), _p(_W(W)), nt, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
        return keys, vic, F, H

    def gang_plan(topo, free, hold, mem, pods, lvl, gang, base=0, W=None):
        topo, free, hold, mem, pods, lvl, gang = (_i32(a) for a in (topo, free, hold, mem, pods, lvl, gang))
        keys, vic = _out(len(pods))
        L.preempt_plan_gang_twin(_p(topo), _p(free), _p(mem), _p(hold), len(free), base, _p(pods), _p(lvl), _p(gang), len(pods),
                                 _p(_W(W)), nt, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
        return keys, vic

    def snapshot(topo, free, hold, mem, pods, lvl, base=0, W=None):
        topo, free, hold, mem, pods, lvl = (_i32(a) for a in (topo, free, hold, mem, pods, lvl))
        keys, vic = _out(len(pods))
        L.preempt_twin_batch(_p(topo), _p(free), _p(mem), _p(hold), len(free), base, _p(pods), _p(lvl), len(pods), _p(_W(W)), 1,
                             _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
        return keys, vic

    return domain_plan, gang_plan, snapshot


def k3_dry_run(topo, free, mem, domain, pods, gang, gd, base=0, W=None):
    """kgpu_place_batch_gang_domain(KGPU_PLACE_DRY_RUN)'s keys, from K3's domain twin."""
    L = gang_domain_libs.twin()
    topo, mem, domain, pods, gang, gd = (_i32(a) for a in (topo, mem, domain, pods, gang, gd))
    f = np.array(free, np.int32, copy=True)
    keys = np.empty(len(pods), np.uint64)
    L.gang_domain_twin_place_batch(_p(topo), _p(f), _p(mem), len(f), base, _p(domain), _p(pods), _p(gang), _p(gd), len(pods),
                                   _p(_W(W)), _p(keys, ctypes.c_uint64))
    return keys


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
def brute_force(snapshot, topo, free, hold, mem, domain, pods, lvl, gang, gd, base=0, W=None):
    """The definition, literally: every member is a single-pod snapshot call on (F, H) with the nodes outside the trial's
    domain masked out (no free GPU, nothing evictable), followed by the update rule; k = 0 takes the domain's lowest node."""
    F, H = _state(free, hold)
    N = len(F)
    keys, vic = np.full(len(pods), NO_FIT, np.uint64), np.zeros(len(pods), np.uint32)

    def one(F, H, q, allowed):
        """member q on (F, H) over the nodes `allowed` (None: all): (key, victims, L, V) after the update, or None."""
        k = int(pods[q, 0])
        if not 0 <= k <= 8:
            return None
        if k == 0:
            n = 0 if allowed is None else int(np.flatnonzero(allowed)[0])
            return np.uint64((base + n) << 8), 0, 0, 0
        Fm, Hm = (F, H) if allowed is None else (np.where(allowed, F, 0), np.where(allowed[:, None], H, -1))
        kk, vv = snapshot(topo, Fm, Hm, mem, pods[q:q + 1], lvl[q:q + 1], base=base, W=W)
        if kk[0] == NO_FIT:
            return None
        n, v = node_of(kk[0], base), int(vv[0])
        levels = [int(H[n, g]) >> 3 for g in range(8) if not (F[n] >> g) & 1 and H[n, g] >= 0 and (v >> (H[n, g] & 7)) & 1]
        S = int(kk[0]) & 0xFF
        R = sum(1 << g for g in range(8) if not (F[n] >> g) & 1 and H[n, g] >= 0 and (v >> (H[n, g] & 7)) & 1)
        F[n] = (int(F[n]) | R) & ~S & 0xFF
        H[n, [g for g in range(8) if ((S | R) >> g) & 1]] = -1
        return kk[0], v, max(levels, default=0), bin(v).count("1")

    def run(members, allowed):
        F2, H2, out = F.copy(), H.copy(), []
        for q in members:
            r = one(F2, H2, q, allowed)
            if r is None:
                return None
            out.append(r)
        return out, F2, H2

    domains = sorted(set(int(d) for d in domain) - {-1})
    p = 0
    while p < len(pods):
        e = p + 1
        while gang[p] != 0 and e < len(pods) and gang[e] == gang[p]:
            e += 1
        res = None
        if gd[p] != 0:
            best = None
            for d in domains:
                r = run(range(p, e), np.asarray(domain) == d)
                if r is not None:
                    score = (max(x[2] for x in r[0]), sum(x[3] for x in r[0]), sum(int(x[0]) >> 40 for x in r[0]), d)
                    if best is None or score < best[0]:
                        best = (score, r)
            res = None if best is None else best[1]
        if res is None and gd[p] != REQ:
            res = run(range(p, e), None)
        if res is not None:
            keys[p:e] = [x[0] for x in res[0]]
            vic[p:e] = [x[1] for x in res[0]]
            F, H = res[1], res[2]
        p = e
    return keys, vic, F, H


def tiny_cluster(seed, N=12, P=30):
    rng = np.random.default_rng(seed)
    topo, _, _ = synth.gen_c4(N=N, P=0, seed=300 + seed)
    free = (rng.integers(0, 256, N) & rng.integers(0, 256, N)).astype(np.int32)
    hold = random_holders(rng, free, levels=6, owners=4)
    domain = rng.integers(-1, 3, N).astype(np.int32)
    pods = synth.make_pods(rng.choice([0, 1, 2, 2, 4, 4, 8, 9], P).astype(np.int32))
    lvl = rng.integers(0, 8, P).astype(np.int32)
    mem = None
    if seed % 2:
        mem = rng.choice([16_384, 32_768, 81_920], (N, 8)).astype(np.int32)
        pods[:, 3] = rng.choice([0, 0, 20_000, 40_000], P)
    gang, gd = random_batch(P, seed, share=0.8)
    return topo, free, hold, mem, domain, pods, lvl, gang, gd


@pytest.mark.parametrize("seed", range(10))
def test_twin_equals_brute_force(plans, seed):
    domain_plan, _, snapshot = plans
    c = tiny_cluster(seed)
    want = brute_force(snapshot, *c, base=5)
    got = domain_plan(*c, base=5)
    for g, w in zip(got, want):
        assert (g == w).all()


def test_tiny_clusters_cover_the_definition(plans):
    """Over the seeds of test_twin_equals_brute_force: REQUIRED gangs placed with victims and failed, PREFERRED gangs
    placed across domains."""
    seen = set()
    for seed in range(10):
        c = tiny_cluster(seed)
        keys, vic, _, _ = plans[0](*c, base=5)
        for a, e in runs(c[7]):
            ok = bool((keys[a:e] != NO_FIT).all())
            one = ok and len({int(c[4][node_of(k, 5)]) for k in keys[a:e] if int(k) & 0xFF}) <= 1
            seen.add((int(c[8][a]), ok, bool((vic[a:e] != 0).any()), one))
    assert (REQ, True, True, True) in seen and (REQ, False, False, False) in seen and (PREF, True, True, False) in seen


# ---- the consequences of the definition, on the twin -------------------------------------------------------------------------
def mid_cluster(seed=3, N=400, P=300, size=8):
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs(N=N, P=P, seed=synth.SEED_PREEMPT_GANGS + seed)
    gd = np.zeros(P, np.int32)
    mode = np.random.default_rng(seed).integers(0, 3, P)
    for a, e in runs(gang):
        gd[a:e] = mode[a]
    return topo, free, hold, None, synth.gen_domains(N, size, seed=seed), pods, lvl, gang, gd


def test_twin_p1_p2_plain_and_one_domain_are_plan_gang(plans):
    domain_plan, gang_plan, _ = plans
    topo, free, hold, mem, domain, pods, lvl, gang, gd = mid_cluster()
    want = gang_plan(topo, free, hold, mem, pods, lvl, gang)
    for g in (None, np.zeros(len(pods), np.int32)):                                      # P1
        got = domain_plan(topo, free, hold, mem, domain, pods, lvl, gang, g)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    for mode in (REQ, PREF):                                                             # P2
        got = domain_plan(topo, free, hold, mem, np.zeros(len(free), np.int32), pods, lvl, gang, np.where(gang != 0, mode, 0))
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all()


@pytest.mark.parametrize("mem", [False, True])
def test_twin_p3_no_eviction_is_k3_domain_dry_run(plans, mem):
    domain_plan, _, _ = plans
    topo, free, hold, _, domain, pods, lvl, gang, gd = mid_cluster(seed=4)
    gm = None
    if mem:
        gm = synth.gen_gpu_memory(len(free), seed=3)
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[np.random.default_rng(1).integers(0, 7, len(pods))]
    domain[::11] = -1
    want = k3_dry_run(topo, free, gm, domain, pods, gang, gd)
    keys, vic, _, _ = domain_plan(topo, free, None, gm, domain, pods, lvl, gang, gd)
    assert (keys == want).all() and (vic == 0).all()
    keys, vic, _, _ = domain_plan(topo, free, hold, gm, domain, pods, np.zeros(len(pods), np.int32), gang, gd)
    assert (keys == want).all() and (vic == 0).all()


def test_twin_p4_p6_required_gangs(plans):
    domain_plan, _, _ = plans
    topo, free, hold, mem, domain, pods, lvl, gang, _ = mid_cluster(seed=5)
    domain[::7] = -1
    gd = np.where(gang != 0, REQ, 0).astype(np.int32)
    keys, vic, _, _ = domain_plan(topo, free, hold, mem, domain, pods, lvl, gang, gd)
    placed, evicting, failed = 0, 0, []
    for a, e in runs(gang):
        if (keys[a:e] == NO_FIT).all():
            assert (vic[a:e] == 0).all()
            failed.append((a, e))
            continue
        placed += 1
        evicting += bool((vic[a:e] != 0).any())
        doms = {int(domain[node_of(k)]) for k in keys[a:e]}                              # P4: victims sit on these nodes
        assert len(doms) == 1 and -1 not in doms
    assert placed > 5 and evicting > 3 and failed
    keep = np.ones(len(pods), bool)                                                      # P6
    for a, e in failed:
        keep[a:e] = False
    k2, v2, _, _ = domain_plan(topo, free, hold, mem, domain, pods[keep], lvl[keep], gang[keep], gd[keep])
    assert (k2 == keys[keep]).all() and (v2 == vic[keep]).all()


def test_twin_p5_preferred_is_required_or_plain(plans):
    domain_plan, gang_plan, _ = plans
    topo, free, hold, mem, domain, pods, lvl, gang, _ = mid_cluster(seed=6, P=200)
    F, H = _state(free, hold)
    kept = fell_back = 0
    for a, e in runs(gang):
        sl, g = slice(a, e), gang[a:e]
        rk, rv, _, _ = domain_plan(topo, F, H, mem, domain, pods[sl], lvl[sl], g, np.full(e - a, REQ, np.int32))
        pk, pv, pF, pH = domain_plan(topo, F, H, mem, domain, pods[sl], lvl[sl], g, np.full(e - a, PREF, np.int32))
        if (rk != NO_FIT).all():
            assert (pk == rk).all() and (pv == rv).all()
            kept += 1
        else:
            gk, gv = gang_plan(topo, F, H, mem, pods[sl], lvl[sl], g)
            assert (pk == gk).all() and (pv == gv).all()
            fell_back += bool((gk != NO_FIT).all())
        F, H = pF, pH
    assert kept > 5 and fell_back > 0


# ---- named cases ------------------------------------------------------------------------------------------------------------
def _topo(shapes):
    return np.stack([synth.shape_matrix(s) for s in shapes])


CHEAP, DEAR = [[8]], [[2, 2], [2, 2]]


def case_required_victims():
    """Full cluster, four domains of two nodes; a level-3 REQUIRED gang of two k = 8 members evicts on both nodes of one
    domain."""
    topo = _topo([CHEAP] * 8)
    hold = np.array([_row(*[(2, 0)] * 4, *[(2, 1)] * 4)] * 8, np.int32)
    pods = synth.make_pods(np.array([8, 8, 2], np.int32))
    return (topo, np.zeros(8, np.int32), hold, None, np.arange(8, dtype=np.int32) // 2, pods, np.array([3, 3, 3], np.int32),
            np.array([1, 1, 0], np.int32), np.array([REQ, REQ, 0], np.int32))


def case_required_nowhere():
    """Domains of two nodes and a REQUIRED gang of three k = 8 members: no domain fits; the plain gang plan would evict
    across domains.  A later solo pod names a victim the gang would have taken."""
    t = list(case_required_victims())
    t[5] = synth.make_pods(np.array([8, 8, 8, 8], np.int32))
    t[6], t[7], t[8] = np.array([3, 3, 3, 3], np.int32), np.array([1, 1, 1, 0], np.int32), np.array([REQ] * 3 + [0], np.int32)
    return tuple(t)


def case_preferred_fallback_fits():
    t = list(case_required_nowhere())
    t[8] = np.where(t[7] != 0, PREF, 0).astype(np.int32)
    return tuple(t)


def case_preferred_fallback_fails():
    """A PREFERRED gang of 9 k = 8 members on 8 nodes: no domain, nor the plain gang plan, fits; the solo pod after it
    still evicts."""
    t = list(case_required_victims())
    t[5] = synth.make_pods(np.array([8] * 10, np.int32))
    t[6], t[7], t[8] = np.full(10, 3, np.int32), np.array([1] * 9 + [0], np.int32), np.array([PREF] * 9 + [0], np.int32)
    return tuple(t)


def case_wins_on_level():
    """Domain 2's nodes cost more but hold level-1 pods, the others level-2 pods: domain 2 wins on L."""
    topo = _topo([CHEAP] * 4 + [DEAR] * 2 + [CHEAP] * 2)
    hold = np.array([_row(*[(2, 0)] * 4, *[(2, 1)] * 4)] * 8, np.int32)
    hold[4:6] = _row(*[(1, 0)] * 4, *[(1, 1)] * 4)
    pods = synth.make_pods(np.array([8, 8], np.int32))
    return (topo, np.zeros(8, np.int32), hold, None, np.arange(8, dtype=np.int32) // 2, pods, np.array([3, 3], np.int32),
            np.ones(2, np.int32), np.full(2, REQ, np.int32))


def case_wins_on_victims():
    """Domain 1's nodes cost more but each holds one 8-GPU pod, the others two 4-GPU pods: domain 1 wins on V."""
    topo = _topo([CHEAP] * 2 + [DEAR] * 2 + [CHEAP] * 2)
    hold = np.array([_row(*[(1, 0)] * 4, *[(1, 1)] * 4)] * 6, np.int32)
    hold[2:4] = _row(*[(1, 0)] * 8)
    pods = synth.make_pods(np.array([8, 8], np.int32))
    return (topo, np.zeros(6, np.int32), hold, None, np.arange(6, dtype=np.int32) // 2, pods, np.array([2, 2], np.int32),
            np.ones(2, np.int32), np.full(2, REQ, np.int32))


def case_tie():
    """Two identical domains: the lower id wins although its nodes have the higher ids."""
    topo = _topo([DEAR] * 4)
    hold = np.array([_row(*[(1, 0)] * 4, *[(1, 1)] * 4)] * 4, np.int32)
    pods = synth.make_pods(np.array([4, 4], np.int32))
    return (topo, np.zeros(4, np.int32), hold, None, np.array([1, 1, 0, 0], np.int32), pods, np.array([2, 2], np.int32),
            np.ones(2, np.int32), np.full(2, REQ, np.int32))


def case_two_members_one_node():
    """Node 0 has 4 free GPUs, node 1 none: two k = 2 members share node 0 without eviction, the third evicts on node 1."""
    topo = _topo([CHEAP] * 4)
    free = np.array([0x0F, 0x00, 0x00, 0x00], np.int32)
    hold = np.array([_row(*[(5, 0)] * 8)] + [_row(*[(1, 0)] * 2, *[(1, 1)] * 2, *[(1, 2)] * 4)] * 3, np.int32)
    pods = synth.make_pods(np.array([2, 2, 2], np.int32))
    return (topo, free, hold, None, np.array([0, 0, 1, 1], np.int32), pods, np.full(3, 3, np.int32), np.ones(3, np.int32),
            np.full(3, REQ, np.int32))


def case_rescore():
    """Node 0 has GPUs 0-3 free and a level-1 pod on 4-7: the first k = 4 member takes 0-3; for the second, node 0 must be
    re-scored in the trial (its table key still says 0-3 are free) and evicts the level-1 pod."""
    topo = _topo([CHEAP] * 4)
    free = np.array([0x0F, 0x00, 0x00, 0x00], np.int32)
    hold = np.array([_row(None, None, None, None, *[(1, 0)] * 4)] + [_row(*[(2, 0)] * 8)] * 3, np.int32)
    pods = synth.make_pods(np.array([4, 4], np.int32))
    return (topo, free, hold, None, np.array([0, 0, 1, 1], np.int32), pods, np.full(2, 3, np.int32), np.ones(2, np.int32),
            np.full(2, REQ, np.int32))


def case_k0_k9():
    topo = _topo([CHEAP] * 6)
    hold = np.array([_row(*[(1, 0)] * 8)] * 6, np.int32)
    free = np.array([0, 0, 0, 0, 0xFF, 0], np.int32)          # domain 1 holds the only free node
    ks = [0, 8, 0, 4, 9, 2]
    gang = [1, 1, 1, 2, 2, 0]
    gd = [REQ] * 3 + [PREF] * 2 + [0]
    return (topo, free, hold, None, np.array([1, 1, 0, 0, 1, 2], np.int32), synth.make_pods(np.array(ks, np.int32)),
            np.full(6, 2, np.int32), np.array(gang, np.int32), np.array(gd, np.int32))


def case_minus_one_nodes():
    """The cheapest victims sit on nodes of no domain: the REQUIRED gang evicts in a domain, a solo pod on a -1 node."""
    topo = _topo([CHEAP] * 6)
    hold = np.array([_row(*[(0, 0)] * 8)] * 2 + [_row(*[(2, 0)] * 8)] * 4, np.int32)
    pods = synth.make_pods(np.array([8, 8, 8], np.int32))
    return (topo, np.zeros(6, np.int32), hold, None, np.array([-1, -1, 0, 0, 1, 1], np.int32), pods, np.full(3, 4, np.int32),
            np.array([1, 1, 0], np.int32), np.array([REQ, REQ, 0], np.int32))


def case_views():
    rng = np.random.default_rng(7)
    N, P = 60, 80
    topo, _, _ = synth.gen_c4(N=N, P=0, seed=8)
    free = (rng.integers(0, 256, N) & rng.integers(0, 256, N)).astype(np.int32)
    hold = random_holders(rng, free, levels=5)
    mem = synth.gen_gpu_memory(N, seed=9)
    pods = synth.make_pods(rng.choice([1, 2, 4, 8], P).astype(np.int32))
    pods[:, 3] = np.array([0, 8_000, 20_000, 40_000], np.int32)[np.arange(P) % 4]
    gang, gd = random_batch(P, 9, share=0.8)
    return topo, free, hold, mem, synth.gen_domains(N, 6, seed=2), pods, rng.integers(0, 6, P).astype(np.int32), gang, gd


def case_chunk():
    """A constrained gang across pod 1024, between plain gangs and solo pods, on three node tiles."""
    rng = np.random.default_rng(11)
    N, P = 300, 1100
    topo, _, _ = synth.gen_c4(N=N, P=0, seed=77)
    free = (rng.integers(0, 256, N) & rng.integers(0, 256, N) & rng.integers(0, 256, N)).astype(np.int32)
    hold = random_holders(rng, free, levels=6)
    pods = synth.make_pods(np.array([1, 2, 3, 5, 8], np.int32)[rng.integers(0, 5, P)])
    lvl = rng.integers(0, 8, P).astype(np.int32)
    gang, gd = np.zeros(P, np.int32), np.zeros(P, np.int32)
    gang[1000:1010] = 1
    gang[1018:1027], gd[1018:1027] = 2, REQ
    pods[1018:1027, 0], lvl[1018:1027] = 2, 7
    gang[1027:1031], gd[1027:1031] = 3, PREF
    gang[1031:1034] = 4
    return topo, free, hold, None, synth.gen_domains(N, 16), pods, lvl, gang, gd


def case_interleaved():
    c = mid_cluster(seed=8, N=300, P=240)
    gang, gd = random_batch(240, 4)
    return c[:7] + (gang, gd)


EMU_CASES = {
    "required_victims": case_required_victims,
    "required_nowhere": case_required_nowhere,
    "preferred_fallback_fits": case_preferred_fallback_fits,
    "preferred_fallback_fails": case_preferred_fallback_fails,
    "wins_on_level": case_wins_on_level,
    "wins_on_victims": case_wins_on_victims,
    "tie": case_tie,
    "two_members_one_node": case_two_members_one_node,
    "rescore": case_rescore,
    "k0_k9": case_k0_k9,
    "minus_one_nodes": case_minus_one_nodes,
    "views": case_views,
    "chunk": case_chunk,
    "interleaved": case_interleaved,
}


def test_cases_are_what_they_claim(plans):
    """Each named case, as the twin plans it."""
    domain_plan, gang_plan, _ = plans

    def go(case):
        c = case()
        return c, domain_plan(*c)

    def doms(c, keys):
        return {int(c[4][node_of(k)]) for k in keys}

    c, (k, v, _, _) = go(case_required_victims)
    assert doms(c, k[:2]) == {0} and (v[:2] != 0).all() and k[2] != NO_FIT
    c, (k, v, _, _) = go(case_required_nowhere)
    blind = gang_plan(c[0], c[1], c[2], None, c[5], c[6], c[7])
    assert (blind[0][:3] != NO_FIT).all() and len(doms(c, blind[0][:3])) > 1
    assert (k[:3] == NO_FIT).all() and (v[:3] == 0).all() and v[3] == 3 and node_of(k[3]) == 0 and blind[1][3] == 3
    assert node_of(blind[0][3]) != 0
    c, (k, v, _, _) = go(case_preferred_fallback_fits)
    assert (k == blind[0]).all() and (v == blind[1]).all()
    c, (k, v, _, _) = go(case_preferred_fallback_fails)
    assert (k[:9] == NO_FIT).all() and (v[:9] == 0).all() and node_of(k[9]) == 0 and v[9] == 3
    c, (k, v, _, _) = go(case_wins_on_level)
    assert doms(c, k) == {2} and (v != 0).all()
    cheap = domain_plan(*(c[:4] + (np.where(c[4] == 0, 0, -1).astype(np.int32),) + c[5:]))[0]
    assert sum(int(x) >> 40 for x in k) > sum(int(x) >> 40 for x in cheap)
    c, (k, v, _, _) = go(case_wins_on_victims)
    assert doms(c, k) == {1} and list(v) == [1, 1]
    cheap = domain_plan(*(c[:4] + (np.where(c[4] == 0, 0, -1).astype(np.int32),) + c[5:]))[0]
    assert sum(int(x) >> 40 for x in k) > sum(int(x) >> 40 for x in cheap)
    c, (k, v, _, _) = go(case_tie)
    assert {node_of(x) for x in k} <= {2, 3} and (v != 0).all()
    c, (k, v, _, _) = go(case_two_members_one_node)
    assert node_of(k[0]) == node_of(k[1]) == 0 and list(v[:2]) == [0, 0] and node_of(k[2]) == 1 and v[2] != 0
    c, (k, v, _, _) = go(case_rescore)
    assert node_of(k[0]) == node_of(k[1]) == 0 and int(k[0]) & 0xFF == 0x0F and int(k[1]) & 0xFF == 0xF0
    assert list(v) == [0, 1]
    c, (k, v, _, _) = go(case_k0_k9)
    assert doms(c, k[:3]) == {1} and node_of(k[0]) == node_of(k[2]) == 0 and int(k[0]) >> 40 == 0 and int(k[0]) & 0xFF == 0
    assert node_of(k[1]) == 4 and v[1] == 0
    assert (k[3:5] == NO_FIT).all() and k[5] != NO_FIT
    c, (k, v, _, _) = go(case_minus_one_nodes)
    assert doms(c, k[:2]) in ({0}, {1}) and c[4][node_of(k[2])] == -1
    c, (k, v, _, _) = go(case_views)
    assert any(gd == REQ and (k[a:e] != NO_FIT).all() and (c[5][a:e, 3] > 0).any() for (a, e), gd in
               ((r, c[8][r[0]]) for r in runs(c[7])))
    c, (k, v, _, _) = go(case_chunk)
    assert (k[1018:1027] != NO_FIT).all() and (v[1018:1027] != 0).any() and len(doms(c, k[1018:1027])) == 1


# ---- the launch plan on the CPU (tests/preempt_plan_domain_emu) ------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return preempt_plan_domain_libs.emu()


def emu_plan(emu, topo, free, hold, mem, domain, pods, lvl, gang, gd, base=0, W=None):
    topo, mem, domain, pods, lvl, gang, gd = (_i32(a) for a in (topo, mem, domain, pods, lvl, gang, gd))
    F, H = _state(free, hold)
    keys, vic = _out(len(pods))
    steps = emu.emu_preempt_plan_gang_domain(_p(topo), _p(F), _p(mem), _p(H), len(F), base, _p(domain), _p(pods), _p(lvl), _p(gang),
                                             _p(gd), len(pods), _p(_W(W)), _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
    assert steps >= 0
    return keys, vic, F, H, steps


@pytest.mark.parametrize("base", [0, 21])
@pytest.mark.parametrize("name", sorted(EMU_CASES))
def test_emulated_plan_matches_twin(emu, plans, name, base):
    c = EMU_CASES[name]()
    keys, vic, F, H, steps = emu_plan(emu, *c, base=base)
    want = plans[0](*c, base=base)
    assert (keys == want[0]).all() and (vic == want[1]).all() and (F == want[2]).all() and (H == want[3]).all()
    gang, gd = c[7], c[8]
    assert steps == sum(1 for a, _ in runs(gang) if gd[a] != 0) > 0


@pytest.mark.parametrize("seed", range(4))
def test_emulated_random_batches(emu, plans, seed):
    rng = np.random.default_rng(seed)
    N, P = int(rng.integers(40, 300)), int(rng.integers(20, 160))
    topo, free, hold, pods, lvl, _ = synth.gen_preempt_gangs(N=N, P=P, seed=synth.SEED_PREEMPT_GANGS + 10 + seed)
    mem = None
    if seed % 2:
        mem = synth.gen_gpu_memory(N, seed=seed)
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[rng.integers(0, 7, P)]
    pods[rng.random(P) < 0.05, 0] = 0
    gang, gd = random_batch(P, seed + 100)
    domain = synth.gen_domains(N, int(rng.choice([1, 4, 8, 32])), seed=seed)
    domain[rng.random(N) < 0.1] = -1
    keys, vic, F, H, _ = emu_plan(emu, topo, free, hold, mem, domain, pods, lvl, gang, gd, base=seed)
    want = plans[0](topo, free, hold, mem, domain, pods, lvl, gang, gd, base=seed)
    assert (keys == want[0]).all() and (vic == want[1]).all() and (F == want[2]).all() and (H == want[3]).all()


# ---- build products --------------------------------------------------------------------------------------------------------
def test_plan_domain_kernels_have_no_local_memory():
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or libkgpu.so missing")
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    lines, found = out.splitlines(), set()
    for i, line in enumerate(lines):
        m = re.search(r"Function _ZN4kgpu\d+(domain_plan_trial|domain_plan_commit)\S*:", line)
        if m:
            found.add(m.group(1))
            assert re.search(r"STACK:0\b", lines[i + 1]) and re.search(r"LOCAL:0\b", lines[i + 1]), lines[i + 1]
    assert found == {"domain_plan_trial", "domain_plan_commit"}


# ---- the device path ---------------------------------------------------------------------------------------------------------
def full_size(use_mem, seed=5):
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs()
    mem = None
    if use_mem:
        mem = synth.gen_gpu_memory(len(free))
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[synth.rand_below(synth.SEED_C6, 14, len(pods), 7)]
    gd = np.zeros(len(pods), np.int32)
    mode = np.random.default_rng(seed).integers(0, 3, len(pods))
    for a, e in runs(gang):
        gd[a:e] = mode[a]
    return topo, free, hold, mem, synth.gen_domains(len(free), 32), pods, lvl, gang, gd


def _scorer(topo, free, hold, mem, domain, base=0):
    from kubegpu_b200.scorer import Scorer
    s = Scorer((0,))
    s.upload_nodes(topo, free, node_id_base=base)
    if mem is not None:
        s.upload_gpu_memory(mem)
    if hold is not None:
        s.upload_holders(hold)
    if domain is not None:
        s.upload_domains(domain)
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("use_mem", [False, True])
def test_device_matches_twin_on_gen_preempt_gangs(plans, use_mem):
    c = full_size(use_mem)
    topo, free, hold, mem, domain, pods, lvl, gang, gd = c
    want_k, want_v, _, _ = plans[0](*c)
    kinds = set()
    for a, e in runs(gang):
        ok = bool((want_k[a:e] != NO_FIT).all())
        kinds.add((int(gd[a]), ok, bool((want_v[a:e] != 0).any()),
                   ok and len({int(domain[node_of(k)]) for k in want_k[a:e]}) == 1))
    assert (REQ, True, True, True) in kinds and (REQ, False, False, False) in kinds
    assert any(m == PREF and ok and not one for m, ok, _, one in kinds)                    # a PREFERRED fallback across domains
    with _scorer(topo, free, hold, mem, domain) as s:
        snap = s.preempt_batch(pods, lvl)
        keys, vic = s.preempt_plan(pods, lvl, gang=gang, gang_domain=gd)
        assert (keys == want_k).all() and (vic == want_v).all()
        assert (s.get_free_masks() == free).all()                                          # the handle's state is untouched
        after = s.preempt_batch(pods, lvl)
        assert (after[0] == snap[0]).all() and (after[1] == snap[1]).all()
        again = s.preempt_plan(pods, lvl, gang=gang, gang_domain=gd)
        assert (again[0] == keys).all() and (again[1] == vic).all()


@pytest.mark.gpu
def test_device_p1_same_result_and_launches():
    topo, free, hold, mem, domain, pods, lvl, gang, _ = full_size(False)
    with _scorer(topo, free, hold, mem, domain, base=7) as s:
        s.preempt_plan(pods, lvl, gang=gang)
        n0 = s.kernel_launches
        want = s.preempt_plan(pods, lvl, gang=gang)
        per_call = s.kernel_launches - n0
        for gd in (None, np.zeros(len(pods), np.int32)):
            n1 = s.kernel_launches
            got = s.preempt_plan(pods, lvl, gang=gang, gang_domain=gd)
            assert (got[0] == want[0]).all() and (got[1] == want[1]).all() and s.kernel_launches - n1 == per_call
        plain = s.preempt_plan(pods, lvl)
        n1 = s.kernel_launches
        got = s.preempt_plan(pods, lvl, gang_domain=np.zeros(len(pods), np.int32))
        assert (got[0] == plain[0]).all() and (got[1] == plain[1]).all() and s.kernel_launches - n1 == per_call


@pytest.mark.gpu
def test_device_p2_to_p5():
    topo, free, hold, _, domain, pods, lvl, gang, _ = full_size(False)
    N = len(free)
    domain[::9] = -1
    with _scorer(topo, free, hold, None, np.zeros(N, np.int32)) as s:
        plain = s.preempt_plan(pods, lvl, gang=gang)
        for mode in (REQ, PREF):                                                           # P2
            got = s.preempt_plan(pods, lvl, gang=gang, gang_domain=np.where(gang != 0, mode, 0))
            assert (got[0] == plain[0]).all() and (got[1] == plain[1]).all()
        s.upload_domains(domain)
        req = np.where(gang != 0, REQ, 0).astype(np.int32)
        keys, vic = s.preempt_plan(pods, lvl, gang=gang, gang_domain=req)                   # P4
        placed = 0
        for a, e in runs(gang):
            if (keys[a:e] != NO_FIT).all():
                placed += 1
                doms = {int(domain[node_of(k)]) for k in keys[a:e]}
                assert len(doms) == 1 and -1 not in doms
        assert placed > 10
        zero = np.zeros(len(pods), np.int32)                                                # P3
        want = s.place_batch(pods, gang=gang, gang_domain=req, dry_run=True)
        k3, v3 = s.preempt_plan(pods, zero, gang=gang, gang_domain=req)
        assert (k3 == want).all() and (v3 == 0).all()
        for a, e in runs(gang)[:30]:                                                        # P5, gang by gang
            g, sl = np.ones(e - a, np.int32), slice(a, e)
            r = s.preempt_plan(pods[sl], lvl[sl], gang=g, gang_domain=np.full(e - a, REQ, np.int32))
            w = r if (r[0] != NO_FIT).all() else s.preempt_plan(pods[sl], lvl[sl], gang=g)
            p = s.preempt_plan(pods[sl], lvl[sl], gang=g, gang_domain=np.full(e - a, PREF, np.int32))
            assert (p[0] == w[0]).all() and (p[1] == w[1]).all()
    with _scorer(topo, free, None, None, domain) as s:                                     # P3 without a holder table
        want = s.place_batch(pods, gang=gang, gang_domain=req, dry_run=True)
        k3, v3 = s.preempt_plan(pods, lvl, gang=gang, gang_domain=req)
        assert (k3 == want).all() and (v3 == 0).all()


@pytest.mark.gpu
def test_device_rejected_inputs():
    from kubegpu_b200.scorer import KgpuError
    topo, free, hold, pods, lvl, _ = synth.gen_preempt_gangs(N=1000, P=6)
    gang = np.array([1, 1, 0, 2, 2, 2], np.int32)
    fn = "kgpu_preempt_plan_gang_domain: "
    cases = [
        (pods, lvl, gang, [1, 1, 0, 3, 3, 3], "gang_domain[3] = 3 is not 0, REQUIRED (1) or PREFERRED (2)"),
        (pods, lvl, gang, [1, 1, 2, 0, 0, 0], "gang_domain[2] = 2 on a pod without a gang"),
        (pods, lvl, gang, [1, 2, 0, 0, 0, 0], "the members of gang 1 disagree on gang_domain"),
        (pods, lvl, None, [1, 0, 0, 0, 0, 0], "gang_domain[0] = 1 on a pod without a gang"),
        (pods, lvl, np.array([3, 3, 0, 4, 3, 3], np.int32), [0] * 6, "gang id 3 appears in two separate runs"),
        (pods, np.array([0, 0, 0, 16, 0, 0], np.int32), gang, [1, 1, 0, 2, 2, 2], "lvl[3] = 16 outside 0..15"),
    ]
    big = synth.make_pods(np.zeros(37_001, np.int32))
    cases.append((big, np.zeros(37_001, np.int32), np.ones(37_001, np.int32), [1] * 37_001,
                  "gang 1 has 37001 members with a domain constraint, more than 37000"))
    many = synth.make_pods(np.ones(8, np.int32))
    many[:, 3] = np.arange(1, 9) * 1000
    cases.append((many, np.ones(8, np.int32), np.ones(8, np.int32), [1] * 8, "more than 7 distinct min_mem values"))
    views = synth.make_pods(np.ones(33, np.int32))
    views[:, 3] = np.repeat(np.array([0, 1000, 2000]), 11)
    cases.append((views, np.tile(np.arange(1, 12), 3).astype(np.int32), np.zeros(33, np.int32), [0] * 33,
                  "more than 32 distinct (level > 0, min_mem) pairs"))
    with _scorer(topo, free, hold, None, synth.gen_domains(1000, 8)) as s:
        want = s.preempt_plan(pods, lvl, gang=gang, gang_domain=np.array([1, 1, 0, 2, 2, 2], np.int32))
        for p, lv, g, gd, msg in cases:
            with pytest.raises(KgpuError) as e:
                s.preempt_plan(p, lv, gang=g, gang_domain=np.array(gd, np.int32))
            assert e.value.code == _lib.ERR_INVALID and fn + msg in str(e.value), str(e.value)
        assert (s.get_free_masks() == free).all()
        got = s.preempt_plan(pods, lvl, gang=gang, gang_domain=np.array([1, 1, 0, 2, 2, 2], np.int32))
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all()


@pytest.mark.gpu
def test_device_two_device_handle_is_refused():
    import torch
    from kubegpu_b200.scorer import KgpuError, Scorer
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    topo, free, hold, pods, lvl, _ = synth.gen_preempt_gangs(N=1000, P=2)
    with Scorer((0, 1)) as s:
        s.upload_nodes(topo, free)
        with pytest.raises(KgpuError) as e:
            s.preempt_plan(pods, lvl, gang=np.ones(2, np.int32), gang_domain=np.ones(2, np.int32))
        assert e.value.code == _lib.ERR_STATE


@pytest.mark.gpu
def test_host_mirror_plans_gangs_in_domains(plans):
    """sched_cli on a full four-node cluster in two racks: preemptgangplan evicts one pod under each rack for a REQUIRED
    two-member gang; preemptdomainplan keeps the gang inside one rack, where it evicts the cheaper victims, and matches the
    twin; a third REQUIRED gang fits in no rack and names nothing."""
    from test_preemption import _node_line
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-s", "-C", ROOT, "kubegpu_b200/lib/kgpu_sched_cli"])
    ids = ["GPU-%02d" % i for i in range(8)]
    names = ["A", "B", "C", "D"]
    racks = {"A": "rack-a", "B": "rack-b", "C": "rack-a", "D": "rack-b"}             # ids: rack-a 0, rack-b 1
    running = [("a1", "A", 1), ("b1", "B", 1), ("c1", "C", 2), ("d1", "D", 2)]
    lines = [_node_line(n, [[4], [4]], ids) for n in names] + ["domain %s %s" % kv for kv in racks.items()]
    for pod, _, prio in running:
        lines += ["pod %s priority=%d run c req=8" % (pod, prio)]
    lines += ["placebatch " + " ".join(p for p, _, _ in running)]
    lines += ["pod g1 priority=3 gang=7 gangdomain=required run c req=8", "pod g2 priority=3 gang=7 gangdomain=required run c req=8",
              "pod h1 priority=3 gang=8 gangdomain=required run c req=8", "pod h2 priority=3 gang=8 gangdomain=required run c req=8",
              "pod h3 priority=3 gang=8 gangdomain=required run c req=8",
              "preemptgangplan g1 g2", "preemptdomainplan g1 g2 h1 h2 h3"]
    got = subprocess.run([CLI], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    blind = got.split("> preemptgangplan g1 g2\n")[1].splitlines()
    dom = got.split("> preemptdomainplan g1 g2 h1 h2 h3\n")[1].splitlines()
    assert blind[0] == "  err=" and dom[0] == "  err=", (blind, dom)
    assert blind[1].endswith("victims=a1") and blind[2].endswith("victims=b1")
    # the twin on the same cluster: node order A..D, every node full, one 8-GPU owner per node
    topo = np.stack([synth.shape_matrix([[4], [4]])] * 4)
    hold = np.array([_row(*[(prio, 0)] * 8) for _, _, prio in running], np.int32)
    pods = synth.make_pods(np.full(5, 8, np.int32))
    want = plans[0](topo, np.zeros(4, np.int32), hold, None, np.array([0, 1, 0, 1], np.int32), pods, np.full(5, 3, np.int32),
                    np.array([7, 7, 8, 8, 8], np.int32), np.full(5, REQ, np.int32))
    assert [node_of(k) for k in want[0][:2]] == [0, 2] and (want[0][2:] == NO_FIT).all()
    for line, k, (pod, victim) in zip(dom[1:3], want[0], (("g1", "a1"), ("g2", "c1"))):
        assert line.startswith("  %s fits=1 " % pod) and " node=%s " % names[node_of(k)] in line and line.endswith("victims=" + victim)
    for line, pod in zip(dom[3:6], ("h1", "h2", "h3")):
        assert line.startswith("  %s fits=0 " % pod) and line.endswith("victims="), line
