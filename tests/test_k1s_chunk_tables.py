"""K1s's per-launch chunk tables on the CPU (the kernels compiled against tests/emu):
sp_prepare_chunks builds every 512-pod chunk's sorted pod table once per launch, and the K1s blocks of a chunk-aligned
work list copy it instead of sorting.  Checked here: both tables against an independent Python layout, the keys of the
prepared path against Oracle B and the in-kernel path, and the work-list rule that decides between them."""
import ctypes

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import synth

CHUNK = 512
DUMMY = 0xFFFF
WEIGHTS = {"default": None, "flat_max": [4095] * 16}


def _p(a, t=ctypes.c_int32):
    return a.ctypes.data_as(ctypes.POINTER(t))


@pytest.fixture(scope="module")
def emu():
    return cpu_libs.emu()


def _pods(P, seed, mem_share=0.3):
    """k in -1..9 (outside 0..8: no launch serves the pod) and min_mem on some pods, a few of them equal."""
    rng = np.random.default_rng(seed)
    pods = synth.make_pods(rng.integers(-1, 10, size=P).astype(np.int32))
    has = rng.random(P) < mem_share
    pods[has, 3] = rng.choice([1024, 16384, 40000, 81920, int(rng.integers(1, 90000))], size=int(has.sum()))
    return pods


def _groups(pods, mem):
    """The chunk's layout as the sort must make it: per k, the (sub-bucket, [(chunk position, multiplier)]) groups in
    order, the bucket offsets (padded to 4), the non-empty mask, and the pods no bucket takes."""
    groups, off, pos, mask = [], [], 0, 0
    k_of, w_of = pods[:, 0], pods[:, 3]
    served = (k_of >= 0) & (k_of <= 8) & ((w_of > 0) == mem)
    sub = ((w_of.astype(np.uint64) * 0x9E3779B1) & 0xFFFFFFFF) >> 30 if mem else np.zeros(len(pods), np.uint64)
    for k in range(9):
        off.append(pos)
        n_k = 0
        for s in range(4 if mem else 1):
            idx = np.flatnonzero(served & (k_of == k) & (sub == s))
            mult = w_of[idx] if mem else np.ones(len(idx), np.int64)
            groups.append((pos + n_k, sorted(zip(idx.tolist(), np.asarray(mult).astype(np.uint32).tolist()))))
            n_k += len(idx)
        mask |= (n_k > 0) << k
        groups.append((pos + n_k, [(DUMMY, 0 if mem else 1)] * (-n_k % 4)))
        pos += (n_k + 3) // 4 * 4
    off.append(pos)
    rest = np.flatnonzero(~served)
    mult = w_of[rest] if mem else k_of[rest]
    groups.append((pos, sorted(zip(rest.tolist(), np.asarray(mult).astype(np.uint32).tolist()))))
    return groups, off, mask


def _check_table(words, pods, mem, npos):
    one = words[:npos].view(np.uint32)
    idx = words[npos:npos + npos // 2].view(np.uint16)
    off = words[npos + npos // 2:npos + npos // 2 + 12]
    groups, want_off, mask = _groups(pods, mem)
    assert off[:10].tolist() == want_off and off[11] == mask
    for start, want in groups:
        got = sorted(zip(idx[start:start + len(want)].tolist(), one[start:start + len(want)].tolist()))
        assert got == want


@pytest.mark.parametrize("P", [513, 1000, 10_000])
@pytest.mark.parametrize("mem", [False, True])
def test_prepared_tables_equal_the_block_sort(emu, P, mem):
    """sp_prepare_chunks and the block's own sort lay every chunk out the same way: buckets k = 0..8 (MEM: sub-bucketed
    by min_mem), each padded with dummy pods to 4 positions, then the pods this launch does not serve."""
    pods = _pods(P, seed=P + mem)
    n_int4, npos = emu.emu_chunk_int4(), emu.emu_chunk_pos()
    chunks = (P + CHUNK - 1) // CHUNK
    prepared = np.zeros((chunks, 4 * n_int4), np.int32)
    sorted_ = np.zeros((chunks, 4 * n_int4), np.int32)
    assert emu.emu_chunk_tables(_p(pods), ctypes.c_int64(P), int(mem), _p(prepared), _p(sorted_)) == chunks
    for c in range(chunks):
        part = pods[c * CHUNK:(c + 1) * CHUNK]
        _check_table(prepared[c], part, mem, npos)
        _check_table(sorted_[c], part, mem, npos)


def _score(emu, topo, free, pods, W, resident, prepare, mem=None, base=0):
    keys = np.zeros(len(pods), np.uint64)
    aligned = emu.emu_score_chunks(_p(topo), _p(free), None if mem is None else _p(mem), ctypes.c_int64(len(free)),
                                   ctypes.c_int64(base), _p(pods), ctypes.c_int64(len(pods)), _p(np.asarray(W, np.int32)),
                                   ctypes.c_int64(resident), int(prepare), _p(keys, ctypes.c_uint64))
    return keys, bool(aligned)


@pytest.mark.parametrize("wname, resident", [("default", 1), ("flat_max", 4)])
def test_prepared_path_keys(emu, wname, resident):
    """On a chunk-aligned work list the K1s blocks take the prepared tables (and skip the k their tile cannot serve);
    the keys equal Oracle B and the blocks' own sort, for pods with and without min_mem.  resident = 1: one item per
    tile over all pods; 4: items that end on chunk boundaries inside the batch as well."""
    from oracle import oracle_b
    W = WEIGHTS[wname] or oracle_b.DEFAULT_WEIGHTS
    topo, free, _ = synth.gen_c2(N=600, P=0, seed=11 + resident)
    free[:40] = 0xFF                                      # a tile of eight-free nodes next to mixed ones
    mem = synth.gen_gpu_memory(len(free), seed=5)
    pods = _pods(1100, seed=resident)
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=7, fast=True, nthreads=4, mem=mem)
    got, aligned = _score(emu, topo, free, pods, W, resident, True, mem=mem, base=7)
    assert aligned
    assert (got == want).all()
    own, _ = _score(emu, topo, free, pods, W, resident, False, mem=mem, base=7)
    assert (own == got).all()


def test_unaligned_list_keeps_the_block_sort(emu):
    """Many resident blocks on a small plane: 32-pod ranges, no prepared tables, the same keys."""
    from oracle import oracle_b
    topo, free, _ = synth.gen_c2(N=300, P=0, seed=3)
    pods = _pods(700, seed=9, mem_share=0.0)
    got, aligned = _score(emu, topo, free, pods, oracle_b.DEFAULT_WEIGHTS, 64, True)
    assert not aligned
    assert (got == oracle_b.score_batch(topo, free, pods, oracle_b.DEFAULT_WEIGHTS, fast=True, nthreads=4)).all()


@pytest.mark.parametrize("tiles, aligned", [(783, True), (80, False)])
def test_work_list_chunk_alignment(emu, tiles, aligned):
    """C2's plane (783 tiles x 20 chunks, 132 SMs x 8 resident blocks) gets whole-chunk ranges; C5's 10k-node shard
    (~80 tiles) keeps 32-pod ranges.  Either way every (tile, pod) cell is covered exactly once."""
    P, resident = 10_000, 132 * 8
    rng = np.random.default_rng(tiles)
    tile_class = np.sort(rng.integers(0, 9, size=tiles).astype(np.uint8))[::-1].copy()
    out = np.zeros((200_000, 4), np.int32)
    flag = ctypes.c_int(-1)
    n = emu.emu_sparse_work(_p(tile_class, ctypes.c_uint8), ctypes.c_int64(tiles), ctypes.c_int64(P), ctypes.c_int64(resident),
                            _p(out), ctypes.c_int64(len(out)), None, ctypes.byref(flag))
    items = out[:n]
    assert flag.value == int(aligned)
    assert (items[:, 3] == 1).all()
    if aligned:
        assert (items[:, 1] % CHUNK == 0).all() and ((items[:, 2] % CHUNK == 0) | (items[:, 2] == P)).all()
    else:
        assert (items[:, 1] % 32 == 0).all() and (items[:, 1] % CHUNK != 0).any()
    cover = np.zeros((tiles, P), np.int8)
    for t, b, e, _ in items:
        assert e > b
        cover[t, b:e] += 1
    assert (cover == 1).all()
