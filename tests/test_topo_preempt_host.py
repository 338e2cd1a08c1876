"""The library's per-node dry run of topology-aware preemption (vct::topo_dry_run in vc_topo.hpp, the code k_evict_dryrun
runs on the device) compiled by g++ into a test shim and compared bit for bit with the exact Python restatement
(tests/topo_kernels_common.py) on random nodes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import topo_kernels_common as K

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostshim", "topo_shim.cpp")
OUT = os.path.join(HERE, "hostshim", "_build", "topo_shim.so")


@pytest.fixture(scope="module")
def shim():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", SRC, "-o", OUT], check=True)
    L = C.CDLL(OUT)
    L.vts_dry_run.argtypes = [C.POINTER(K.EhTopoArgs)]
    return L


@pytest.mark.parametrize("block", range(6))
def test_dry_run_matches_the_restatement(shim, block):
    """Random nodes (0-300 pods, R 2-16, integer and non-integer requests, random voter tiers, simulate hooks on / off,
    indexed and unindexed pod names mixed in one job): success, victims in list order and the four scores identical."""
    hits = 0
    for seed in range(block * 25, block * 25 + 25):
        rng = np.random.default_rng(seed)
        I = K.random_instance(rng, int(rng.integers(1, 80)), int(rng.integers(2, 17)), max_pods=int(rng.choice([12, 300])),
                              non_integer=seed % 2 == 1)
        a, out = K.to_args(I)
        assert shim.vts_dry_run(C.byref(a)) == 0
        hits += K.check_dry_run(I, out, range(I["N"]))
    assert hits >= 20


def test_victim_order_is_the_heap_not_a_sort(shim):
    """util.LessFn is not a strict weak order when indexed and unindexed pod names meet (A(idx 1, ts 5) < B(idx 2, ts 1) <
    C(no idx, ts 3) < A). Three such victims of one job on one node, all needed: the list is the Go heap's pop order,
    reversed by the reprieve, as the restatement's container/heap produces it."""
    I = K.random_instance(np.random.default_rng(0), 1, 2, max_pods=3, heavy=0)
    RT = 3
    I.update(RT=RT, rt_off=np.array([0, 3], np.int32), rt_idx=np.arange(3, dtype=np.int32),
             rt_req=np.ones((2, RT)), rt_has=np.zeros(RT, np.uint32),
             rt_flags=np.full(RT, abi_flags(), np.uint32), rt_uid=np.arange(RT, dtype=np.uint32),
             rt_job=np.ones(RT, np.int32), rt_prio=np.zeros(RT, np.int32), rt_pod_prio=np.array([1, 2, 3], np.int32),
             rt_podidx=np.array([1, 2, -1], np.int64), rt_ts=np.array([5, 1, 3], np.int64),
             rt_start=np.zeros(RT, np.int64), rt_evicted=np.zeros(RT, np.uint8),
             idle=np.zeros((2, 1)), rel=np.zeros((2, 1)), pip=np.zeros((2, 1)), pred=np.ones(1, np.uint8),
             req=np.array([3.0, 3.0]), has=0, intra=0, sim_update=0, sim_alloc=0, task_order_prio=0)
    I["j_queue"][:] = 0
    I["queue"] = 0
    I["j_min"][:] = 0
    I["j_ready"][:] = 10
    I["plugin"] = np.array([K.VOTERS[0]], np.int32)
    I["tier"], I["enabled"], I["n_plugins"] = np.zeros(1, np.int32), np.array([K.abi.VC_EN_PREEMPTABLE], np.uint32), 1
    a, out = K.to_args(I)
    assert shim.vts_dry_run(C.byref(a)) == 0
    assert K.check_dry_run(I, out, [0]) == 1
    assert list(out["victims"][:3]) == K.dry_run(I, 0)[0]


def abi_flags():
    return K.abi.VC_RT_PREEMPTABLE | K.abi.VC_RT_RUNNING
