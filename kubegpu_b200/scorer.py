"""Handle wrapper over the C ABI: what bench.py and the GPU tests drive.

Mirrors the call sequence a Go ``DeviceScheduler`` host makes through cgo
(INTEGRATION.md): create -> upload_nodes (AddNode for the whole cluster) ->
score_batch per scheduling cycle -> update_node / remove_node as the cluster changes.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence

import numpy as np

from . import _lib


class KgpuError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("libkgpu error %d: %s" % (code, msg))
        self.code = code


def _i32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.int32)


class Scorer:
    """One libkgpu handle (``kgpu_t``) on one or more CUDA devices."""

    def __init__(self, devices: Sequence[int] = (0,)):
        self._L = _lib.load()
        self._h = ctypes.c_void_p()
        devs = (ctypes.c_int * len(devices))(*devices)
        rc = self._L.kgpu_create(devs, len(devices), ctypes.byref(self._h))
        if rc != _lib.OK:
            self._h = ctypes.c_void_p()
            raise KgpuError(rc, (self._L.kgpu_last_error(None) or b"").decode())
        self.devices = tuple(devices)

    # -- plumbing ---------------------------------------------------------------
    def _check(self, rc: int) -> None:
        if rc != _lib.OK:
            raise KgpuError(rc, (self._L.kgpu_last_error(self._h) or b"").decode())

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            self._L.kgpu_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # -- configuration ----------------------------------------------------------
    def set_weights(self, w) -> None:
        w = _i32(w)
        if w.size != 16:
            raise ValueError("weights must have 16 entries")
        self._check(self._L.kgpu_set_weights(self._h, w.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))))

    def get_weights(self) -> np.ndarray:
        w = np.zeros(16, dtype=np.int32)
        self._check(self._L.kgpu_get_weights(self._h, w.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))))
        return w

    def set_variant(self, variant: int) -> None:
        self._check(self._L.kgpu_set_variant(self._h, int(variant)))

    # -- node array (AddNode / RemoveNode side) -----------------------------------
    def upload_nodes(self, topo, free_mask, node_id_base: int = 0) -> None:
        topo, free_mask = _i32(topo), _i32(free_mask)
        n = free_mask.shape[0]
        if topo.size != 64 * n:
            raise ValueError("topo must be [N,64] for N = len(free_mask)")
        p32 = ctypes.POINTER(ctypes.c_int32)
        self._check(self._L.kgpu_upload_nodes(self._h, topo.ctypes.data_as(p32), free_mask.ctypes.data_as(p32),
                                              n, int(node_id_base)))

    def upload_gpu_memory(self, mem_mib) -> None:
        """mem_mib[N,8]: MiB per GPU slot; pods' min_mem_mib (pods[:,3]) is checked against it."""
        mem = _i32(mem_mib)
        if mem.size != 8 * self.num_nodes:
            raise ValueError("mem_mib must be [N,8]")
        self._check(self._L.kgpu_upload_gpu_memory(self._h, mem.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), self.num_nodes))

    def update_gpu_memory(self, idx: int, mem_mib) -> None:
        mem = _i32(mem_mib)
        if mem.size != 8:
            raise ValueError("mem_mib must have 8 entries")
        self._check(self._L.kgpu_update_gpu_memory(self._h, int(idx), mem.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))))

    def update_node(self, idx: int, topo, free_mask: int) -> None:
        topo = _i32(topo)
        if topo.size != 64:
            raise ValueError("topo must have 64 entries")
        self._check(self._L.kgpu_update_node(self._h, int(idx), topo.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                             int(free_mask)))

    def set_free_mask(self, idx: int, free_mask: int) -> None:
        self._check(self._L.kgpu_set_free_mask(self._h, int(idx), int(free_mask)))

    def set_free_masks(self, idx, free_masks) -> None:
        """Batched state change (a cycle's Take/Return): one copy + one kernel; last entry wins on duplicates."""
        idx = np.ascontiguousarray(idx, dtype=np.int64)
        fm = _i32(free_masks)
        if idx.shape[0] != fm.shape[0]:
            raise ValueError("idx and free_masks must have the same length")
        self._check(self._L.kgpu_set_free_masks(self._h, idx.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                                fm.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), idx.shape[0]))

    def build_fit_table(self) -> None:
        self._check(self._L.kgpu_build_fit_table(self._h))

    def fit_lookup(self, node_idx: int, k: int) -> int:
        """(cost << 8 | mask) of node node_idx for k GPUs from the handle's host-side (node, k) table, or 0xFFFFFFFF."""
        out = ctypes.c_uint32()
        self._check(self._L.kgpu_fit_lookup(self._h, int(node_idx), int(k), ctypes.byref(out)))
        return int(out.value)

    @property
    def last_upload_ms(self) -> float:
        return float(self._L.kgpu_last_upload_ms(self._h))

    def remove_node(self, idx: int) -> None:
        self._check(self._L.kgpu_remove_node(self._h, int(idx)))

    @property
    def num_nodes(self) -> int:
        return int(self._L.kgpu_num_nodes(self._h))

    # -- scoring ------------------------------------------------------------------
    def score_batch(self, pods, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Host buffers in, host buffers out (the end-to-end call)."""
        pods = _i32(pods)
        P = pods.size // 4
        if out is None:
            out = np.empty(P, dtype=np.uint64)
        self._check(self._L.kgpu_score_batch(self._h, pods.ctypes.data, P, out.ctypes.data))
        return out

    def place_batch(self, pods, out: Optional[np.ndarray] = None, dry_run: bool = False, gang=None,
                    gang_domain=None, gang_level=None) -> np.ndarray:
        """Stateful sequential placement: pods in order, each takes its GPUs (device free masks change).
        dry_run: conflict-free proposals on a scratch copy of the masks, the handle's state is untouched.
        gang: int32[P] gang ids, 0 = the pod is on its own.  A run of consecutive pods with the same nonzero id
        is placed all or nothing: if a member does not fit, the members before it give their GPUs back and the
        whole gang gets NO_FIT.  An id in two separate runs raises KgpuError (ERR_INVALID).
        gang_domain: int32[P], 0 = no constraint, 1 (GANG_DOMAIN_REQUIRED) = the gang is placed inside one domain of
        upload_domains or not at all, 2 (GANG_DOMAIN_PREFERRED) = inside one domain if one fits, else as a plain gang.
        Nonzero only on gang members, the same for every member of a gang (include/kgpu.h has the definition).
        gang_level: int32[P], the highest level of a multi-level domain table a constrained gang may span (0 on other
        pods, the same for every member): the gang takes the lowest level 0..gang_level with a domain that fits, then
        the cheapest domain there.  None = all 0, which is the level-0 placement."""
        pods = _i32(pods)
        P = pods.size // 4
        if out is None:
            out = np.empty(P, dtype=np.uint64)
        flags = _lib.PLACE_DRY_RUN if dry_run else 0
        if gang is None and gang_domain is None and gang_level is None:
            self._check(self._L.kgpu_place_batch_ex(self._h, pods.ctypes.data, P, out.ctypes.data, flags))
            return out
        if gang is not None:
            gang = _i32(gang)
            if gang.size != P:
                raise ValueError("gang must hold one id per pod")
        if gang_domain is None and gang_level is None:
            self._check(self._L.kgpu_place_batch_gang(self._h, pods.ctypes.data, gang.ctypes.data, P, out.ctypes.data, flags))
            return out
        if gang_domain is not None:
            gang_domain = _i32(gang_domain)
            if gang_domain.size != P:
                raise ValueError("gang_domain must hold one value per pod")
        g = None if gang is None else gang.ctypes.data
        gd = None if gang_domain is None else gang_domain.ctypes.data
        if gang_level is None:
            self._check(self._L.kgpu_place_batch_gang_domain(self._h, pods.ctypes.data, g, gd, P,
                                                             out.ctypes.data, flags))
            return out
        gang_level = _i32(gang_level)
        if gang_level.size != P:
            raise ValueError("gang_level must hold one value per pod")
        self._check(self._L.kgpu_place_batch_gang_levels(self._h, pods.ctypes.data, g, gd,
                                                         gang_level.ctypes.data, P, out.ctypes.data, flags))
        return out

    def upload_domains(self, domain) -> None:
        """domain[N]: each node's network domain, -1 (none) or 0..N-1 (the nodes under one leaf switch, one scalable
        unit or one NVLink Switch domain).  domain[L, N]: L nested levels (1..MAX_DOMAIN_LEVELS), level 0 the finest
        (a rack), each level's ids separate; the nodes of one level-l domain share one level-(l + 1) domain
        (kgpu_upload_domain_levels has the rules).  Until the first upload, and after upload_nodes, every node is in
        none."""
        dom = _i32(domain)
        if dom.ndim not in (1, 2) or dom.shape[-1] != self.num_nodes:
            raise ValueError("domain must hold one value per node (per level)")
        ptr = dom.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
        if dom.ndim == 1:
            self._check(self._L.kgpu_upload_domains(self._h, ptr, dom.size))
        else:
            self._check(self._L.kgpu_upload_domain_levels(self._h, ptr, dom.shape[0], dom.shape[1]))

    # -- preemption (PostFilter) -----------------------------------------------------
    def upload_holders(self, holders) -> None:
        """holders[N,8]: per GPU slot -1 (not evictable) or level << 3 | owner (level 0..15, owner 0..7); GPUs of one
        owner belong to one running pod and carry one level.  Entries of free GPUs are ignored."""
        hold = _i32(holders)
        if hold.size != 8 * self.num_nodes:
            raise ValueError("holders must be [N,8]")
        self._check(self._L.kgpu_upload_holders(self._h, hold.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), self.num_nodes))

    def set_holders(self, idx, holders) -> None:
        """Replace the holder rows of nodes idx (one copy); the last row wins on duplicates."""
        idx = np.ascontiguousarray(idx, dtype=np.int64)
        hold = _i32(holders)
        if hold.size != 8 * idx.shape[0]:
            raise ValueError("holders must be [len(idx),8]")
        self._check(self._L.kgpu_set_holders(self._h, idx.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                             hold.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), idx.shape[0]))

    def preempt_batch(self, pods, lvl):
        """(keys uint64[P], victims uint32[P]): for each pod the best placement when running pods of a lower level
        (lvl[p], 0..15) may be evicted, smallest (max victim level, victim count, cost, node, mask) first.  A pod that
        fits without eviction gets its score_batch key and victims 0; victims bit o = owner o of the key's node."""
        pods, lvl = _i32(pods), _i32(lvl)
        P = pods.size // 4
        if lvl.size != P:
            raise ValueError("lvl must hold one level per pod")
        keys = np.empty(P, dtype=np.uint64)
        victims = np.empty(P, dtype=np.uint32)
        self._check(self._L.kgpu_preempt_batch(self._h, pods.ctypes.data, lvl.ctypes.data, P, keys.ctypes.data,
                                               victims.ctypes.data))
        return keys, victims

    def preempt_plan(self, pods, lvl, gang=None, gang_domain=None):
        """(keys uint64[P], victims uint32[P]) as preempt_batch, but conflict-free: pods are taken in order, each on the
        state the pods before it leave (their GPUs taken, their victims' GPUs free, neither evictable again).  Victim
        sets are disjoint.  Dry run: the handle's masks and holder table are untouched.  Pass pods in priority order.
        gang: int32[P] gang ids as for place_batch.  A gang's members evict and take all together or not at all: if a
        member misses, the members before it are undone (their victims are running pods again for later pods) and the
        whole gang gets NO_FIT and victims 0.  An id in two separate runs raises KgpuError (ERR_INVALID).
        gang_domain: int32[P] as for place_batch.  A REQUIRED gang evicts and takes its GPUs inside the one domain of
        upload_domains whose trial plan is best in (max victim level, victim count, summed cost, domain id), or gets
        NO_FIT; a PREFERRED gang falls back to the plain gang plan (include/kgpu.h has the definition)."""
        pods, lvl = _i32(pods), _i32(lvl)
        P = pods.size // 4
        if lvl.size != P:
            raise ValueError("lvl must hold one level per pod")
        keys = np.empty(P, dtype=np.uint64)
        victims = np.empty(P, dtype=np.uint32)
        if gang_domain is not None:
            gang = None if gang is None else _i32(gang)
            gang_domain = _i32(gang_domain)
            if (gang is not None and gang.size != P) or gang_domain.size != P:
                raise ValueError("gang and gang_domain must hold one value per pod")
            self._check(self._L.kgpu_preempt_plan_gang_domain(self._h, pods.ctypes.data, lvl.ctypes.data,
                                                              None if gang is None else gang.ctypes.data,
                                                              gang_domain.ctypes.data, P, keys.ctypes.data, victims.ctypes.data))
            return keys, victims
        if gang is None:
            self._check(self._L.kgpu_preempt_plan(self._h, pods.ctypes.data, lvl.ctypes.data, P, keys.ctypes.data,
                                                  victims.ctypes.data))
            return keys, victims
        gang = _i32(gang)
        if gang.size != P:
            raise ValueError("gang must hold one id per pod")
        self._check(self._L.kgpu_preempt_plan_gang(self._h, pods.ctypes.data, lvl.ctypes.data, gang.ctypes.data, P,
                                                   keys.ctypes.data, victims.ctypes.data))
        return keys, victims

    def get_free_masks(self) -> np.ndarray:
        out = np.empty(self.num_nodes, dtype=np.int32)
        self._check(self._L.kgpu_get_free_masks(self._h, out.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), out.shape[0]))
        return out

    def score_pairs(self, node_idx, ks, min_mem=None) -> np.ndarray:
        """Per-pair query: (cost << 8 | mask) of node node_idx[i] for k = ks[i] (and min_mem[i] MiB per
        GPU if given), or 0xFFFFFFFF."""
        node_idx = np.ascontiguousarray(node_idx, dtype=np.int64)
        ks = _i32(ks)
        mm = None if min_mem is None else _i32(min_mem)
        out = np.empty(node_idx.shape[0], dtype=np.uint32)
        self._check(self._L.kgpu_score_pairs(self._h, node_idx.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                             ks.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                             None if mm is None else mm.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                             node_idx.shape[0],
                                             out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32))))
        return out

    def score_batch_ptr(self, pods_addr: int, P: int, out_addr: int) -> None:
        """Same call on raw host addresses (e.g. pinned torch tensors' data_ptr())."""
        self._check(self._L.kgpu_score_batch(self._h, pods_addr, int(P), out_addr))

    def score_batch_device(self, d_pods_addr: int, P: int, d_keys_addr: int, stream: int = 0, batch_flags: int = 0) -> None:
        """Device buffers, enqueued on `stream` (cudaStream_t as int, 0 = the CUDA default stream).
        batch_flags: _lib.BATCH_NO_MIN_MEM promises that no pod carries min_mem_mib > 0."""
        if batch_flags:
            self._check(self._L.kgpu_score_batch_device_ex(self._h, d_pods_addr, int(P), d_keys_addr, stream or None, int(batch_flags)))
        else:
            self._check(self._L.kgpu_score_batch_device(self._h, d_pods_addr, int(P), d_keys_addr, stream or None))

    def reduce_shards_device(self, d_gathered_addr: int, G: int, P: int, d_out_addr: int, stream: int = 0) -> None:
        self._check(self._L.kgpu_reduce_shards_device(self._h, d_gathered_addr, int(G), int(P), d_out_addr,
                                                      stream or None))

    # ---- peer-memory key exchange (EXPERIMENTAL; one process per GPU) -------------------------
    def exchange_init(self, world: int, rank: int, max_pods: int) -> bytes:
        """Allocate this rank's result/flag memory; returns the 64-byte IPC handle to all-gather."""
        buf = ctypes.create_string_buffer(_lib.IPC_HANDLE_BYTES)
        self._check(self._L.kgpu_exchange_init(self._h, int(world), int(rank), int(max_pods), buf))
        return bytes(buf.raw)

    def exchange_connect(self, handles) -> None:
        """handles: the world's IPC handles in rank order (list of 64-byte strings)."""
        blob = b"".join(bytes(x) for x in handles)
        if len(blob) % _lib.IPC_HANDLE_BYTES:
            raise ValueError("every handle must be %d bytes" % _lib.IPC_HANDLE_BYTES)
        self._check(self._L.kgpu_exchange_connect(self._h, ctypes.c_char_p(blob)))

    def score_batch_exchange(self, d_pods_addr: int, P: int, stream: int = 0, batch_flags: int = 0) -> int:
        """K1 on the local shard + push/sync over peer memory; returns the DEVICE address of the global keys
        (uint64[P], owned by the handle, valid until the next-but-one call)."""
        out = ctypes.c_void_p()
        self._check(self._L.kgpu_score_batch_exchange(self._h, d_pods_addr, int(P), ctypes.byref(out), stream or None, int(batch_flags)))
        return int(out.value or 0)

    def exchange_barrier(self, stream: int = 0) -> None:
        """Device-side barrier of the ranks (the exchange kernel with no pods), enqueued on `stream`."""
        self._check(self._L.kgpu_exchange_barrier(self._h, stream or None))

    @property
    def kernel_launches(self) -> int:
        return int(self._L.kgpu_kernel_launches(self._h))

    @property
    def last_kernel_ms(self) -> float:
        return float(self._L.kgpu_last_kernel_ms(self._h))


def unpack_key(key: int):
    """(cost, node_id, gpu_mask) or None for KGPU_NO_FIT."""
    key = int(key)
    if key == _lib.NO_FIT:
        return None
    return key >> 40, (key >> 8) & 0xFFFFFFFF, key & 0xFF
