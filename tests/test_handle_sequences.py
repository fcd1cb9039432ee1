"""A libkgpu handle driven through long seeded sequences of calls, checked after every call against HandleModel, a host-side
model of the state include/kgpu.h documents (node array, free masks, GPU memory, holder table, weights, variant, node-id
base) and nothing more.  The handle keeps caches that some calls invalidate and others refresh in place: the K1s order
(stale while fewer than n / 200 nodes changed), its compacted records, the host-side (node, k) fit table and the work list,
which is cached by the pod count alone.  The sequences mix the calls that touch those caches, so a cache left stale by
any combination of them shows up as a key that differs from the references:
    score_batch         class_keys (test_memory_aware_at_scale): Oracle B once per (k, requirement) class
    fit_lookup / score_pairs                oracle_b.node_key on the node's (eligible) free mask
    place_batch[_gang] (dry run or not)     oracle_b.place_batch / the gang twin
    preempt_batch / preempt_plan[_gang]     the preemption twins
A failing check names the seed, the step and the last five calls, so the log alone reproduces it."""
import ctypes
import os
import time

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import _lib, synth
from test_memory_aware_at_scale import class_keys

pytestmark = pytest.mark.gpu

NO_FIT = np.uint64(_lib.NO_FIT)
INT32_MAX = 2**31 - 1
NTHREADS = os.cpu_count() or 1
POD_COUNTS = (1, 4, 5, 64, 65, 300, 512, 513, 1000, 2048)
VARIANTS = (_lib.VARIANT_AUTO, _lib.VARIANT_WARP_PER_PAIR, _lib.VARIANT_LANE_PER_NODE, _lib.VARIANT_MEMO_BY_K,
            _lib.VARIANT_TILE_MEMO, _lib.VARIANT_SPARSE)
DEFAULT_W = np.array([64, 32, 16, 8, 4, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0], np.int32)
# the largest byte-key table and the smallest general-key one (launch_plan.h: byte_keys), and the all-tie table
WEIGHTS = (DEFAULT_W, np.array([2340 - 7 * i for i in range(16)], np.int32), np.array([2341 - 7 * i for i in range(16)], np.int32),
           np.zeros(16, np.int32))
REQUIREMENTS = (0, 16_384, 20_000, 81_921)                  # no requirement, a class value, between classes, above one
ALL_NVLINK = np.where(np.eye(8, dtype=bool), 0, 12).astype(np.int32).reshape(64)
ALL_FIFTEEN = np.full(64, 15, np.int32)


def _p(a, t=ctypes.c_int32):
    return a.ctypes.data_as(ctypes.POINTER(t))


def _opt(a, t=ctypes.c_int32):
    return None if a is None else _p(np.ascontiguousarray(a, dtype=np.int32), t)


def node_of(key, base):
    return (int(key) >> 8 & 0xFFFFFFFF) - base


class HandleModel:
    """What a handle holds according to include/kgpu.h: every call's documented effect on it, nothing about caches."""

    def __init__(self, topo, free, base=0):
        self.upload_nodes(topo, free, base)
        self.W = DEFAULT_W.copy()
        self.variant = _lib.VARIANT_AUTO

    @property
    def n(self):
        return len(self.free)

    def upload_nodes(self, topo, free, base=0):            # memory back to unlimited, holder table back to all -1
        self.topo, self.free, self.base = np.array(topo, np.int32), np.array(free, np.int32), int(base)
        self.mem = self.hold = None

    def upload_gpu_memory(self, mem):
        self.mem = np.array(mem, np.int32)

    def update_gpu_memory(self, i, row):
        if self.mem is None:
            self.mem = np.full((self.n, 8), INT32_MAX, np.int32)
        self.mem[i] = row

    def update_node(self, i, row, mask):
        self.topo[i], self.free[i] = row, mask

    def set_free_masks(self, idx, masks):                   # the last entry of a node wins
        for i, m in zip(idx, masks):
            self.free[i] = m

    def set_holders(self, idx, rows):
        if self.hold is None:
            self.hold = np.full((self.n, 8), -1, np.int32)
        for i, r in zip(idx, rows):
            self.hold[i] = r

    def eligible(self, i, need):
        if self.mem is None or need <= 0:
            return int(self.free[i])
        return int(self.free[i]) & sum(1 << g for g in range(8) if self.mem[i][g] >= need)


class References:
    """Oracle B and the CPU twins, called on the model's state."""

    def __init__(self, oracle_b):
        self.ob = oracle_b
        self.pre = cpu_libs.twin("preempt_plan_gang")
        self.k3 = cpu_libs.twin("gang")

    def score(self, m, pods):
        return class_keys(self.ob, m.topo, m.free, pods, m.W, m.base, m.mem)

    def node_key(self, m, i, k, need=0):
        return self.ob.node_key(m.topo[i], m.eligible(i, need), k, m.W)

    def place(self, m, pods, gang=None):
        """(keys, free masks after)"""
        if gang is None:
            return self.ob.place_batch(m.topo, m.free, pods, m.W, node_id_base=m.base, mem=m.mem)
        F = m.free.copy()
        keys = np.empty(len(pods), np.uint64)
        self.k3.gang_twin_place_batch(_p(m.topo), _p(F), _opt(m.mem), m.n, m.base, _p(pods), _opt(gang), len(pods), _p(m.W),
                                      _p(keys, ctypes.c_uint64))
        return keys, F

    def preempt(self, m, fn, pods, lvl, gang=None):
        keys, vic = np.empty(len(pods), np.uint64), np.empty(len(pods), np.uint32)
        args = [_p(m.topo), _p(m.free), _opt(m.mem), _opt(m.hold), m.n, m.base, _p(pods), _p(lvl)]
        if gang is not None:
            args.append(_opt(gang))
        getattr(self.pre, fn)(*args, len(pods), _p(m.W), NTHREADS, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
        return keys, vic


class Sequence:
    """One seeded run: the handle, the model, the call log and the checks."""

    def __init__(self, scorer, refs, seed, N, multi=False):
        self.s, self.refs, self.seed, self.multi = scorer, refs, seed, multi
        self.rng = np.random.default_rng(seed)
        self.step = 0
        self.log = []
        self.touched = []
        self.fixed_P = False
        self.evictions = 0                                         # pods the preemption references let evict
        self.P = int(self.rng.choice(POD_COUNTS))
        self.pods = self.make_pods(self.P)
        topo, free = self.cluster(N)
        self.call("upload_nodes(n=%d, base=0)" % N, lambda: scorer.upload_nodes(topo, free))
        self.m = HandleModel(topo, free)

    # -- bookkeeping ----------------------------------------------------------------------------------------------------
    def call(self, what, fn):
        self.log.append("step %d: %s" % (self.step, what))
        return fn()

    def fail(self, what):
        raise AssertionError("seed %d, step %d: %s\nlast calls:\n  %s" % (self.seed, self.step, what, "\n  ".join(self.log[-5:])))

    def expect_keys(self, got, want, pods, what):
        bad = np.flatnonzero(np.asarray(got) != np.asarray(want))
        if len(bad):
            i = int(bad[0])
            self.fail("%s: %d of %d keys differ; first at pod %d (k %d, min_mem %d): got %x, want %x"
                      % (what, len(bad), len(want), i, pods[i, 0], pods[i, 3], int(got[i]), int(want[i])))

    # -- inputs ---------------------------------------------------------------------------------------------------------
    def cluster(self, N):
        """gen_c2's four shapes (cost ties everywhere) with a few all-NVLink nodes, node 0 and the last node included.  An
        eighth of the GPUs are free, so that pods of 8 GPUs fit nowhere until masks change and preemption has work."""
        topo, free, _ = synth.gen_c2(N=N, P=0, seed=int(self.rng.integers(1 << 30)))
        topo = topo.copy()
        free = (free & self.rng.integers(0, 256, size=N) & self.rng.integers(0, 256, size=N)).astype(np.int32)
        nv = np.concatenate([[0, N - 1], self.rng.integers(0, N, size=8)])
        topo[nv] = ALL_NVLINK
        return topo, free

    def make_pods(self, P):
        """k mostly 1..8, with 0 and out-of-range k; a third of the pods carry a requirement from REQUIREMENTS."""
        k = self.rng.integers(1, 9, size=P)
        u = self.rng.random(P)
        k[u < 0.05] = 0
        k[(u >= 0.05) & (u < 0.08)] = 9
        pods = synth.make_pods(k.astype(np.int32))
        has = self.rng.random(P) < 0.35
        pods[has, 3] = self.rng.choice(REQUIREMENTS, size=int(has.sum()))
        return pods

    def some_nodes(self, cnt):
        """Random nodes, the ends of the array and of a multi-device handle's shards, and recently touched nodes."""
        n = self.m.n
        edges = [0, n - 1]
        if self.multi:
            per = (n + 1) // 2
            edges += [per - 1, min(per, n - 1)]
        pool = np.concatenate([self.rng.integers(0, n, size=cnt), edges, self.touched[-16:]]).astype(np.int64)
        return np.clip(pool, 0, n - 1)

    def holder_rows(self, cnt):
        """Owner g // 2 on GPU g (four pods of two GPUs per node) at a level 0..3 per owner, some GPUs not evictable."""
        lv = self.rng.integers(0, 4, size=(cnt, 4))
        rows = (np.repeat(lv, 2, axis=1) << 3) | (np.arange(8) // 2)
        rows[self.rng.random((cnt, 8)) < 0.2] = -1
        return rows.astype(np.int32)

    def memory(self, n):
        return synth.gen_gpu_memory(n, seed=int(self.rng.integers(1 << 30)))

    # -- mutations --------------------------------------------------------------------------------------------------------
    def mutate(self, kind):
        s, m, rng = self.s, self.m, self.rng
        if kind == "set_free_masks":
            cnt = int(rng.choice([1, 8, 150, 250, 600]))
            idx = self.some_nodes(cnt)
            idx = np.concatenate([idx, idx[: cnt // 4]])          # duplicates: the last entry of a node wins
            masks = rng.choice([0, 0xFF, 0x0F, 0x80, 0x01], size=len(idx)).astype(np.int32)
            rnd = rng.random(len(idx)) < 0.6
            masks[rnd] = rng.integers(0, 256, size=int(rnd.sum()))
            self.call("set_free_masks(%d entries)" % len(idx), lambda: s.set_free_masks(idx, masks))
            m.set_free_masks(idx, masks)
            self.touched += list(idx[-8:])
        elif kind == "set_free_mask":
            i, mk = int(self.some_nodes(1)[0]), int(rng.choice([0, 0xFF, int(rng.integers(0, 256))]))
            self.call("set_free_mask(%d, %#x)" % (i, mk), lambda: s.set_free_mask(i, mk))
            m.free[i] = mk
            self.touched.append(i)
        elif kind == "remove_node":
            i = int(self.some_nodes(1)[0])
            self.call("remove_node(%d)" % i, lambda: s.remove_node(i))
            m.free[i] = 0
            self.touched.append(i)
        elif kind == "update_node":
            i = int(self.some_nodes(2)[rng.integers(0, 2)])
            choice = int(rng.integers(0, 4))
            row = (ALL_NVLINK, ALL_FIFTEEN, m.topo[int(rng.integers(0, m.n))].copy(), m.topo[i].copy())[choice]
            mk = int(rng.choice([0xFF, 0, int(rng.integers(0, 256))]))
            self.call("update_node(%d, topology %d, %#x)" % (i, choice, mk), lambda: s.update_node(i, row, mk))
            m.update_node(i, row, mk)
            self.touched.append(i)
        elif kind == "upload_gpu_memory":
            mem = self.memory(m.n)
            self.call("upload_gpu_memory", lambda: s.upload_gpu_memory(mem))
            m.upload_gpu_memory(mem)
        elif kind == "update_gpu_memory":
            i = int(self.some_nodes(1)[0])
            row = rng.choice(list(synth.GPU_MEM_CLASSES_MIB) + [0, 20_000, INT32_MAX], size=8).astype(np.int32)
            self.call("update_gpu_memory(%d, %s)" % (i, row.tolist()), lambda: s.update_gpu_memory(i, row))
            m.update_gpu_memory(i, row)
            self.touched.append(i)
        elif kind == "set_weights":
            j = int(rng.integers(0, len(WEIGHTS)))
            self.call("set_weights(table %d)" % j, lambda: s.set_weights(WEIGHTS[j]))
            m.W = WEIGHTS[j].copy()
        elif kind == "set_variant":
            v = int(rng.choice(VARIANTS))
            self.call("set_variant(%d)" % v, lambda: s.set_variant(v))
            m.variant = v
        elif kind in ("place_batch", "place_batch_gang"):
            self.commit_place(gang=kind == "place_batch_gang")
        elif kind == "upload_holders":
            rows = self.holder_rows(m.n)
            self.call("upload_holders", lambda: s.upload_holders(rows))
            m.hold = rows
        elif kind == "set_holders":
            idx = self.some_nodes(40)
            rows = self.holder_rows(len(idx))
            self.call("set_holders(%d rows)" % len(idx), lambda: s.set_holders(idx, rows))
            m.set_holders(idx, rows)
        elif kind == "upload_nodes":
            n = max(129, m.n + int(rng.choice([-1, 1])) * int(rng.integers(1, 4000)))
            self.upload(n, int(rng.choice([0, 7, 2**32 - 1 - n])))
        else:
            raise ValueError(kind)

    def upload(self, n, base):
        topo, free = self.cluster(n)
        self.call("upload_nodes(n=%d, base=%d)" % (n, base), lambda: self.s.upload_nodes(topo, free, node_id_base=base))
        self.m.upload_nodes(topo, free, base)
        self.touched = []

    def small_batch(self, P=24):
        pods = self.make_pods(P)
        pods[:, 0] = np.clip(pods[:, 0], 0, 8)
        return pods

    def commit_place(self, gang):
        """A committed place_batch[_gang]; on a SPARSE handle the next score_batch re-sorts the order (build_order: 3
        launches, compact_nodes over every slot: 1)."""
        s, m = self.s, self.m
        pods = self.small_batch()
        gid = np.where(np.arange(len(pods)) < 12, np.arange(len(pods)) // 4 + 1, 0).astype(np.int32) if gang else None
        sparse = m.variant == _lib.VARIANT_SPARSE
        if sparse:
            self.score_launches()                                  # brings the caches up to date
            steady = self.score_launches()
        want, free_after = self.refs.place(m, pods, gid)
        got = self.call("place_batch(P=%d, gang=%s)" % (len(pods), gang), lambda: s.place_batch(pods, gang=gid))
        self.expect_keys(got, want, pods, "committed place_batch")
        m.free = free_after
        self.touched += [node_of(k, m.base) for k in want if k != NO_FIT][:8]
        if sparse:
            after = self.score_launches(check=True)
            if after != steady + 4:
                self.fail("the score_batch after a committed place_batch made %d launches, want %d + 4 (re-sort)" % (after, steady))

    # -- checks -----------------------------------------------------------------------------------------------------------
    def score_launches(self, check=False):
        """Launches of one score_batch of the current batch, its keys checked if asked."""
        l0 = self.s.kernel_launches
        got = self.call("score_batch(P=%d)" % self.P, lambda: self.s.score_batch(self.pods))
        launches = self.s.kernel_launches - l0
        if check:
            self.expect_keys(got, self.refs.score(self.m, self.pods), self.pods, "score_batch P=%d" % self.P)
        return launches

    def check_state(self):
        s, m, rng = self.s, self.m, self.rng
        if self.step % 4 == 0 and not self.fixed_P:                # one P for several steps: the work list is cached by P
            self.P = int(rng.choice(POD_COUNTS))
            self.pods = self.make_pods(self.P)
        self.score_launches(check=True)
        got = self.call("get_free_masks", s.get_free_masks)
        if not (got == m.free).all():
            i = int(np.flatnonzero(got != m.free)[0])
            self.fail("get_free_masks: node %d has %#x, want %#x" % (i, int(got[i]), int(m.free[i])))
        nodes = self.some_nodes(12)
        ks = rng.integers(0, 9, size=len(nodes))
        self.call("fit_lookup x %d" % len(nodes), lambda: (s.fit_lookup(0, 1), s.fit_lookup(m.n - 1, 1)))
        l0 = s.kernel_launches                                     # every shard's table is valid now: lookups never launch
        for i, k in zip(nodes, ks):
            got, want = s.fit_lookup(int(i), int(k)), self.refs.node_key(m, int(i), int(k))
            if got != want:
                self.fail("fit_lookup(%d, %d) = %x, want %x" % (i, k, got, want))
        if s.kernel_launches != l0:
            self.fail("fit_lookup launched %d kernels on a valid table" % (s.kernel_launches - l0))
        need = rng.choice(REQUIREMENTS, size=len(nodes)).astype(np.int32)
        for mm in (None, need):
            got = self.call("score_pairs(%d, min_mem=%s)" % (len(nodes), mm is not None), lambda: s.score_pairs(nodes, ks, mm))
            want = [self.refs.node_key(m, int(i), int(k), 0 if mm is None else int(mm[j])) for j, (i, k) in enumerate(zip(nodes, ks))]
            if [int(x) for x in got] != want:
                j = next(j for j in range(len(want)) if int(got[j]) != want[j])
                self.fail("score_pairs(min_mem=%s) pair %d (node %d, k %d): %x, want %x"
                          % (mm is not None, j, nodes[j], ks[j], int(got[j]), want[j]))

    def check_dry_runs(self):
        """A dry-run place_batch, preempt_batch, preempt_plan and preempt_plan_gang against their references; none of them
        changes the handle: the masks stay, and the next score_batch makes as many launches as the one before."""
        s, m = self.s, self.m
        self.score_launches()
        steady = self.score_launches()
        pods = self.small_batch()
        want, _ = self.refs.place(m, pods)
        got = self.call("place_batch(P=%d, dry_run)" % len(pods), lambda: s.place_batch(pods, dry_run=True))
        self.expect_keys(got, want, pods, "dry-run place_batch")
        pods = pods.copy()
        pods[:, 0] = self.rng.choice([1, 2, 4, 8, 8], size=len(pods))      # most pods of 8 GPUs can only fit by evicting
        lvl = self.rng.integers(0, 5, size=len(pods)).astype(np.int32)
        gid = np.where(np.arange(len(pods)) < 9, np.arange(len(pods)) // 3 + 1, 0).astype(np.int32)
        for fn, call, gang in (("preempt_twin_batch", lambda: s.preempt_batch(pods, lvl), None),
                               ("preempt_plan_twin", lambda: s.preempt_plan(pods, lvl), None),
                               ("preempt_plan_gang_twin", lambda: s.preempt_plan(pods, lvl, gang=gid), gid)):
            got_k, got_v = self.call(fn.replace("_twin", ""), call)
            want_k, want_v = self.refs.preempt(m, fn, pods, lvl, gang)
            self.expect_keys(got_k, want_k, pods, fn)
            self.evictions += int((want_v != 0).sum())
            if not (got_v == want_v).all():
                i = int(np.flatnonzero(got_v != want_v)[0])
                self.fail("%s: victims of pod %d are %#x, want %#x" % (fn, i, int(got_v[i]), int(want_v[i])))
        if not (s.get_free_masks() == m.free).all():
            self.fail("a dry run changed the free masks")
        after = self.score_launches(check=True)
        if after != steady:
            self.fail("score_batch made %d launches after the dry runs, %d before them" % (after, steady))

    def check_resort_threshold(self):
        """SPARSE: after a committed place_batch and one score_batch the order is fresh; n // 400 changed nodes leave it
        alone, n // 200 + 1 of them make the next score_batch re-sort."""
        s, m = self.s, self.m
        self.call("set_variant(SPARSE)", lambda: s.set_variant(_lib.VARIANT_SPARSE))
        m.variant = _lib.VARIANT_SPARSE
        self.commit_place(gang=False)
        steady = self.score_launches()
        nodes = self.rng.permutation(m.n)[: m.n // 200 + 1].astype(np.int64)
        first, second = nodes[: m.n // 400], nodes[m.n // 400:]
        for part, extra in ((first, 0), (second, 4)):
            masks = (m.free[part] ^ 0x11).astype(np.int32)
            self.call("set_free_masks(%d distinct nodes)" % len(part), lambda: s.set_free_masks(part, masks))
            m.set_free_masks(part, masks)
            got = self.score_launches(check=True)
            if got != steady + extra:
                self.fail("score_batch after %d changed nodes of %d made %d launches, want %d" % (
                    len(part) if extra == 0 else len(nodes), m.n, got, steady + extra))


SINGLE_KINDS = ("set_free_masks", "set_free_masks", "set_free_mask", "remove_node", "update_node", "update_node",
                "upload_gpu_memory", "update_gpu_memory", "set_weights", "set_variant", "set_variant", "place_batch",
                "place_batch_gang", "upload_holders", "set_holders", "upload_nodes")
MULTI_KINDS = ("set_free_masks", "set_free_masks", "set_free_mask", "remove_node", "update_node", "update_node",
               "upload_gpu_memory", "update_gpu_memory", "set_weights", "set_variant", "upload_nodes")


def run_sequence(scorer, refs, seed, N, steps, multi=False):
    t0 = time.perf_counter()
    seq = Sequence(scorer, refs, seed, N, multi)
    kinds = MULTI_KINDS if multi else SINGLE_KINDS
    seq.check_state()
    for step in range(1, steps + 1):
        seq.step = step
        kind = kinds[int(seq.rng.integers(0, len(kinds)))]
        seq.mutate(kind)
        seq.check_state()
        if not multi and step % 6 == 0:
            seq.check_dry_runs()
        if not multi and step % 20 == 10:
            seq.check_resort_threshold()
    print("seed %d: %d steps, %d nodes at the start and %d at the end, %d evicting pods, %.1f s"
          % (seed, steps, N, seq.m.n, seq.evictions, time.perf_counter() - t0))


@pytest.fixture(scope="module")
def refs(oracle_b):
    return References(oracle_b)


def test_fixed_transitions(refs):
    """The transitions a random sequence reaches only by chance, in a fixed order on a SPARSE handle with one pod count:
      - the cached work list across uploads of more and then fewer nodes (more / fewer tiles), and across a re-sort;
      - set_weights on a stale order (one compact over the old order, keys in the new weights), both key formats;
      - holders uploaded, then a new node array: its holder table is all -1 again (preempt_batch == score_batch);
      - a committed place_batch followed by row patches of the fit table (set_free_masks, update_node)."""
    from kubegpu_b200.scorer import Scorer
    with Scorer((0,)) as s:
        seq = Sequence(s, refs, 100, 2_000)                       # the work list for 2048 pods is built on 16 tiles
        seq.step = 1
        seq.fixed_P, seq.P = True, 2048
        seq.pods = seq.make_pods(2048)
        seq.call("set_variant(SPARSE)", lambda: s.set_variant(_lib.VARIANT_SPARSE))
        seq.m.variant = _lib.VARIANT_SPARSE
        seq.check_state()
        for n in (30_001, 12_000):
            seq.step += 1
            seq.upload(n, 3)
            seq.check_state()
        seq.step += 1
        seq.commit_place(gang=False)
        seq.check_state()
        for w in (1, 2, 0):                                       # byte keys, general keys, back; each on a stale order
            seq.step += 1
            seq.mutate("set_free_masks")
            seq.mutate("update_node")
            seq.call("set_weights(table %d)" % w, lambda: s.set_weights(WEIGHTS[w]))
            seq.m.W = WEIGHTS[w].copy()
            seq.check_state()
        seq.step += 1
        seq.mutate("upload_holders")
        seq.check_dry_runs()
        seq.upload(8_000, 0)                                      # fewer nodes: the table's memory is reused
        seq.check_dry_runs()
        pods = seq.small_batch(64)
        pods[::2, 0] = 8
        keys, vic = seq.call("preempt_batch(level 15)", lambda: s.preempt_batch(pods, np.full(64, 15, np.int32)))
        if (vic != 0).any() or not (keys == s.score_batch(pods)).all():
            seq.fail("preempt_batch after a new node array evicts or differs from score_batch")
        seq.step += 1
        seq.mutate("place_batch")
        for kind in ("set_free_masks", "update_node", "set_free_mask", "remove_node"):
            seq.mutate(kind)
            seq.check_state()


@pytest.mark.parametrize("seed,N,steps",[(1, 40_000, 40), (2, 40_000, 40), (3, 40_000, 40), (4, 129, 60)])
def test_handle_sequence(refs, seed, N, steps):
    from kubegpu_b200.scorer import Scorer
    with Scorer((0,)) as s:
        run_sequence(s, refs, seed, N, steps)


def test_handle_sequence_two_devices(refs):
    """The calls a multi-device handle takes (masks, node and memory updates, fit_lookup, score_pairs, score_batch) are
    routed to the shard of each index; N is odd so the shards are uneven, and the nodes next to the split are updated."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from kubegpu_b200.scorer import Scorer
    with Scorer((0, 1)) as s:
        run_sequence(s, refs, 5, 40_001, 40, multi=True)
