"""The handle's device and pinned buffers (kubegpu_b200/csrc/buffer.h): every allocation of libkgpu goes through the
one owning buffer type, each buffer with its own capacity.  CPU: no raw allocation or free outside that type.  GPU:
call sequences that grow one scratch buffer next to others, or re-upload a larger cluster after a batch with many
memory classes, answer bit-exact against Oracle B and the preemption twin."""
import ctypes
import os
import re

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "kubegpu_b200", "csrc")
NO_FIT = np.uint64(0xFFFFFFFFFFFFFFFF)
RAW_CALLS = ("cudaMalloc(", "cudaFree(", "cudaMallocHost(", "cudaFreeHost(")


def _p(a, t=ctypes.c_int32):
    return a.ctypes.data_as(ctypes.POINTER(t))


def _without_buffer_type(text):
    """text with the body of `class Buffer` cut out."""
    m = re.search(r"\bclass Buffer\b[^;{]*\{", text)
    assert m, "no class Buffer"
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        i += 1
    return text[:m.start()] + text[i:]


def test_allocations_only_in_buffer_type():
    with open(os.path.join(CSRC, "buffer.h")) as f:
        header = f.read()
    with open(os.path.join(CSRC, "kgpu.cu")) as f:
        lib = f.read()
    assert all(c in header for c in ("cudaMalloc(", "cudaFree(", "cudaMallocHost(", "cudaFreeHost("))
    for name, text in (("buffer.h", _without_buffer_type(header)), ("kgpu.cu", lib)):
        for n, line in enumerate(text.splitlines(), 1):
            assert not any(c in line for c in RAW_CALLS), "%s:%d allocates or frees outside the buffer type: %s" % (name, n, line.strip())


# ---- the device path -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def preempt_twin():
    """preempt(topo, free, pods, lvl, hold=None, mem=None) -> (keys, victims): tests/preempt_twin built with the oracle."""
    from oracle import oracle_b
    L = cpu_libs.twin("preempt")
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)

    def preempt(topo, free, pods, lvl, hold=None, mem=None):
        topo, free, pods, lvl = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, lvl))
        opt = [None if a is None else _p(np.ascontiguousarray(a, dtype=np.int32)) for a in (mem, hold)]
        keys = np.empty(len(pods), dtype=np.uint64)
        vic = np.empty(len(pods), dtype=np.uint32)
        L.preempt_twin_batch(_p(topo), _p(free), opt[0], opt[1], len(free), 0, _p(pods), _p(lvl), len(pods), _p(W),
                             os.cpu_count() or 1, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
        return keys, vic
    return preempt


def _eligible(mem, i, m):
    return sum(1 << g for g in range(8) if mem[i][g] >= m)


def _pair_keys(ob, topo, free, idx, ks, mm=None, mem=None):
    if mm is None:
        return [ob.node_key(topo[i], int(free[i]), int(k)) for i, k in zip(idx, ks)]
    return [ob.node_key(topo[i], int(free[i]) & _eligible(mem, i, int(m)), int(k)) for i, k, m in zip(idx, ks, mm)]


def _holders(rng, n):
    """A valid holder table: each GPU to one of 8 owners, one level 0..3 per owner, a tenth of the entries -1."""
    own = rng.integers(0, 8, size=(n, 8))
    hold = (np.take_along_axis(rng.integers(0, 4, size=(n, 8)), own, axis=1) << 3 | own).astype(np.int32)
    hold[rng.random((n, 8)) < 0.1] = -1
    return hold


def _runs(gang):
    out, p = [], 0
    while p < len(gang):
        e = p + 1
        while e < len(gang) and gang[e] == gang[p]:
            e += 1
        if gang[p] != 0:
            out.append((int(gang[p]), p, e))
        p = e
    return out


def _by_deletion(ob, topo, free, pods, gang, keys):
    """Oracle B's placement of the batch without the gangs that failed in `keys`, NO_FIT for their pods."""
    failed = np.isin(gang, [g for g, a, e in _runs(gang) if (keys[a:e] == NO_FIT).any()])
    kk, ff = ob.place_batch(topo, free, pods[~failed])
    want = np.full(len(pods), NO_FIT, dtype=np.uint64)
    want[~failed] = kk
    return want, ff


def _check_preempt(s, twin, rng, topo, free, mem=None):
    """Upload a holder table for the current masks and check preempt_batch's keys and victims."""
    hold = _holders(rng, len(free))
    pods = synth.make_pods(np.array([1, 2, 4, 8], np.int32)[rng.integers(0, 4, size=600)])
    lvl = rng.integers(0, 5, size=600).astype(np.int32)
    want_k, want_v = twin(topo, free, pods, lvl, hold=hold, mem=mem)
    s.upload_holders(hold)
    keys, vic = s.preempt_batch(pods, lvl)
    assert (keys == want_k).all() and (vic == want_v).all()
    assert (vic != 0).any()


@pytest.mark.gpu
def test_dry_run_after_query_growth(oracle_b):
    """A dry run, score_pairs with min_mem on enough pairs to grow the query buffers, a second dry run, then a commit:
    the dry-run scratch is left alone by the query buffers' growth."""
    from kubegpu_b200.scorer import Scorer
    topo, free, mem, pods = synth.gen_c6(N=2000, P=500)
    want, wf = oracle_b.place_batch(topo, free, pods, mem=mem)
    rng = np.random.default_rng(3)
    idx = rng.integers(0, len(free), size=400).astype(np.int64)
    ks = rng.integers(1, 9, size=400).astype(np.int32)
    mm = np.array([8_000, 20_000, 40_000, 100_000], np.int32)[rng.integers(0, 4, size=400)]
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_gpu_memory(mem)
        assert (s.place_batch(pods, dry_run=True) == want).all()
        assert s.score_pairs(idx, ks, mm).tolist() == _pair_keys(oracle_b, topo, free, idx, ks, mm, mem)
        assert (s.place_batch(pods, dry_run=True) == want).all()
        assert (s.get_free_masks() == free).all()
        assert (s.place_batch(pods) == want).all() and (s.get_free_masks() == wf).all()
        s.close()


@pytest.mark.gpu
def test_place_tables_after_growth(oracle_b, preempt_twin):
    """1000 nodes and a batch with 7 distinct min_mem values (8 views), then a re-upload of 5000 nodes and a batch
    without min_mem: the half tables follow the node count.  On both arrays also dry runs, the fit table, gangs and
    preemption, so that every buffer sized by the node count is used past its first size."""
    from kubegpu_b200.scorer import Scorer
    rng = np.random.default_rng(11)
    topo, free, mem, _ = synth.gen_c6(N=1000, P=0)
    pods = synth.make_pods(rng.integers(1, 9, size=400).astype(np.int32))
    classes = np.array([0, 1_000, 10_000, 16_384, 20_000, 32_768, 50_000, 81_920], np.int32)
    pods[:, 3] = classes[np.arange(400) % 8]
    want, wf = oracle_b.place_batch(topo, free, pods, mem=mem)
    idx = rng.integers(0, 1000, size=300).astype(np.int64)
    ks = rng.integers(1, 9, size=300).astype(np.int32)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_gpu_memory(mem)
        assert (s.place_batch(pods, dry_run=True) == want).all() and (s.get_free_masks() == free).all()
        assert (s.place_batch(pods) == want).all() and (s.get_free_masks() == wf).all()
        assert s.score_pairs(idx, ks).tolist() == _pair_keys(oracle_b, topo, wf, idx, ks)
        _check_preempt(s, preempt_twin, rng, topo, wf, mem=mem)

        topo, free, gpods, gang = synth.gen_gangs(N=5000, P=2000)
        assert (gpods[:, 3] == 0).all()
        s.upload_nodes(topo, free)
        plain, gp, gg = gpods[:800], gpods[800:], gang[800:]
        want, wf = oracle_b.place_batch(topo, free, plain)
        assert (s.place_batch(plain) == want).all() and (s.get_free_masks() == wf).all()
        dry = s.place_batch(gp, dry_run=True, gang=gg)
        assert (s.get_free_masks() == wf).all()
        got = s.place_batch(gp, gang=gg)
        want, wf = _by_deletion(oracle_b, topo, wf, gp, gg, got)
        assert (got == dry).all() and (got == want).all() and (s.get_free_masks() == wf).all()
        assert (got != NO_FIT).any() and (got == NO_FIT).any()      # some gangs placed, some failed
        idx = rng.integers(0, 5000, size=300).astype(np.int64)
        assert s.score_pairs(idx, ks).tolist() == _pair_keys(oracle_b, topo, wf, idx, ks)
        _check_preempt(s, preempt_twin, rng, topo, wf)
