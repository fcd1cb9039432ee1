"""CPU-only checks on the SASS of the headline K1s instantiation (score_pairs_sparse<PER_PAIR, !MEM, BYTE_KEYS>,
the kernel that scores C2): its (K, F) bucket loops keep local memory out, and their instruction count per
(warp, pod) on C2's mix stays at the level the four-pod trips reach."""
import os
import shutil
import sys

import pytest

from kubegpu_b200 import _lib

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import k1s_issue_model  # noqa: E402


@pytest.fixture(scope="module")
def loops():
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or libkgpu.so missing")
    return k1s_issue_model.bucket_loops(_lib.LIB_PATH, k1s_issue_model.HEADLINE)[1]


def test_bucket_loops_local_memory(loops):
    assert len(loops) == 30                            # (K, F) loops: K = 0, 1 one each, K >= 2: F = K..8
    assert sum(l[3] for l in loops) <= 5


def test_bucket_loops_trip_widths(loops):
    widths = sorted({l[2] for l in loops[1:]})         # (the k = 0 loop shares one REDUX between its pods)
    assert widths == [2, 4]
    assert loops[1][2] == 4                            # k = 1: nothing but per-pod overhead, four pods per trip


def test_model_instructions_per_warp_pod_c2():
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or libkgpu.so missing")
    _, per_pod, _ = k1s_issue_model.per_pod(_lib.LIB_PATH, ks=(1, 2, 4, 8))
    assert per_pod <= 10.0
