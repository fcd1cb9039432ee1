"""Multi-GPU paths on the GPU box (need >= 2 devices; skipped otherwise):
 - the single-process handle kgpu_create(devs, n>1): shards + NCCL all-gather + K2 inside libkgpu
 - per-pair queries routed to the right shard."""
import numpy as np
import pytest

from kubegpu_b200 import synth

pytestmark = pytest.mark.gpu


def _ndev():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("G", [2, 4, 8])
def test_multi_device_handle_matches_oracle(oracle_b, G):
    if _ndev() < G:
        pytest.skip("needs %d GPUs" % G)
    from kubegpu_b200.scorer import Scorer
    topo, free, pods = synth.gen_c4(N=50_001, P=321)
    want = oracle_b.score_batch(topo, free, pods, node_id_base=17, fast=True, nthreads=8)
    with Scorer(tuple(range(G))) as s:
        s.upload_nodes(topo, free, node_id_base=17)
        assert s.num_nodes == 50_001
        assert (s.score_batch(pods) == want).all()
        # per-pair queries land on whichever shard owns the node
        idx = np.array([0, 1, 25_000, 25_001, 49_999, 50_000], dtype=np.int64)
        ks = np.array([1, 2, 3, 4, 5, 8], dtype=np.int32)
        got = s.score_pairs(idx, ks)
        for i, k, g in zip(idx, ks, got):
            assert int(g) == oracle_b.node_key(topo[i], int(free[i]), int(k))
        # update a node on the last shard and rescore
        topo2, free2 = topo.copy(), free.copy()
        topo2[50_000] = 9
        free2[50_000] = 0xFF
        s.update_node(50_000, topo2[50_000], 0xFF)
        assert (s.score_batch(pods) == oracle_b.score_batch(topo2, free2, pods, node_id_base=17, fast=True, nthreads=8)).all()


def test_sequential_placement_on_two_devices_in_one_process(oracle_b):
    """K3 opts in to its dynamic shared memory per device: single-device handles on devices 0 and 1 of one process both
    place (plain and gang batches) and match the oracle."""
    if _ndev() < 2:
        pytest.skip("needs 2 GPUs")
    from kubegpu_b200.scorer import Scorer
    topo, free, pods = synth.gen_c4(N=3000, P=200, seed=5)
    alone = np.zeros(len(pods), dtype=np.int32)             # gang ids 0: every pod on its own, the plain placement
    want, want_free = oracle_b.place_batch(topo, free.copy(), pods)
    with Scorer((0,)) as a, Scorer((1,)) as b:
        for s in (a, b):
            s.upload_nodes(topo, free)
            assert (s.place_batch(pods, dry_run=True, gang=alone) == want).all()
            assert (s.place_batch(pods) == want).all() and (s.get_free_masks() == want_free).all()


def test_torchrun_bench_keys_equal_single_gpu(tmp_path):
    """The one-process-per-GPU path of bench.py (torch.distributed NCCL all-gather + K2): the final
    keys at N=2 must be the very same bits as at N=1 (SURVEY.md 8(e): result independent of G)."""
    import json
    import os
    import subprocess
    import sys
    if _ndev() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")

    def line(cmd):
        out = subprocess.run(cmd, cwd=root, env=env, capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-2000:]
        return json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])

    one = line([sys.executable, "bench.py", "--steps", "2", "--warmup", "3", "--no-cpu-baseline", "--no-variants"])
    two = line([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                "--master-port", "29533", "bench.py", "--gpus", "2", "--steps", "2", "--warmup", "3"])
    assert one["n_gpus"] == 1 and two["n_gpus"] == 2
    assert one["keys_sha256_12"] == two["keys_sha256_12"]
    assert two["config"]["nodes"] == 100_000 and two["scaling"] == "strong"


def test_torchrun_push_exchange_keys_equal_single_gpu():
    """The peer-memory exchange (kgpu_score_batch_exchange: stores into every rank's slots over NVLink + flag barrier +
    local minimum, one kernel) must give the very same keys as one GPU and as the NCCL all-gather + K2 path."""
    import json
    import os
    import subprocess
    import sys
    if _ndev() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")

    def line(cmd):
        out = subprocess.run(cmd, cwd=root, env=env, capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-2000:]
        return json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])

    one = line([sys.executable, "bench.py", "--steps", "3", "--warmup", "3", "--no-cpu-baseline", "--no-variants"])
    one_push = line([sys.executable, "bench.py", "--steps", "3", "--warmup", "3", "--no-cpu-baseline", "--no-variants", "--exchange", "push"])
    two = line([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                "--master-port", "29534", "bench.py", "--gpus", "2", "--steps", "5", "--warmup", "3", "--exchange", "push"])
    assert one["keys_sha256_12"] == one_push["keys_sha256_12"] == two["keys_sha256_12"]
    assert "peer-memory" in two["config"]["parallelism"]
