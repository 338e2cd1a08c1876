"""The library's host-side hdrf logic (vc_hdrf.hpp: tree construction and evaluation; the hdrf comparator in
vch::backfill_pick) compiled by g++ into a test shim and compared with the hdrf oracle (tools/hdrf_oracle) on the CPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import hdrf_common as H
from volcano_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostshim", "hdrf_shim.cpp")
OUT = os.path.join(HERE, "hostshim", "_build", "hdrf_shim.so")
_dp, _i32p = C.POINTER(C.c_double), C.POINTER(C.c_int32)


@pytest.fixture(scope="module")
def shim():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", SRC, "-o", OUT], check=True)
    return C.CDLL(OUT)


def _tree(shim, snap):
    hd = snap.hdrf()
    total = snap.n_allocatable.sum(axis=1)
    total_has = sum(1 << d for d in range(2, snap.R)) if snap.N else 0
    share = np.zeros(snap.J)
    for j in range(snap.J):  # drf.calculateShare over dims with total >= 0.1
        share[j] = max([(snap.j_allocated[d, j] / total[d]) for d in range(snap.R) if total[d] >= 0.1] + [0.0])
    off = np.zeros(snap.Q + 1, np.int32)
    n = 64 * (snap.Q + 1)
    sh, w, sat = np.zeros(n), np.zeros(n), np.zeros(n, np.int32)
    why = C.create_string_buffer(256)
    m = shim.vhh_tree(snap.R, snap.J, snap.Q, snap.j_queue.ctypes.data_as(_i32p), C.byref(hd), total.ctypes.data_as(_dp),
                      C.c_uint32(total_has), np.ascontiguousarray(snap.j_allocated).ctypes.data_as(_dp),
                      share.ctypes.data_as(_dp), off.ctypes.data_as(_i32p), sh.ctypes.data_as(_dp), w.ctypes.data_as(_dp),
                      sat.ctypes.data_as(_i32p), why, 256)
    return m, off, sh, w, sat, why.value.decode()


@pytest.mark.parametrize("cfg,seed", [("tiny", s) for s in range(8)] + [("small", s) for s in range(4)])
def test_tree_at_open_matches_the_oracle(shim, cfg, seed):
    """vch::hdrf_build + the replica's full refresh: every node on every queue's path has the oracle's share (bit for
    bit), weight and saturation at session open."""
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg, seed)
    hier, wts = H.random_tree(snap, np.random.default_rng(50 + seed))
    m, off, sh, w, sat, why = _tree(shim, snap)
    assert m > 0, why
    o = H.HdrfOracle(snap, hier, wts)
    has_job = set(int(q) for q in snap.j_queue)
    checked = 0
    for q in range(snap.Q):
        if q not in has_job:
            continue
        for lvl in range(off[q + 1] - off[q]):
            s, wt, st, _ = o.node(q, lvl)
            i = off[q] + lvl
            assert (sh[i], w[i], bool(sat[i])) == (s, wt, st), (q, lvl)
            checked += 1
    assert checked >= snap.Q


def test_refusals_in_the_library(shim):
    """The library's tree construction refuses what the reference crashes on (weights shorter than the path)."""
    from volcano_b200.synth import make_snapshot, total_request
    snap = make_snapshot("tiny", 1)
    snap.set_hdrf(["root/a/b"] * snap.Q, ["1/2"] * snap.Q, total_request(snap))
    m, *_, why = _tree(shim, snap)
    assert m == -1 and "weights" in why


@pytest.mark.parametrize("cfg,seed", [("tiny_bf", s) for s in range(6)] + [("small_bf", s) for s in range(3)])
def test_backfill_pick_order_matches_the_oracle(shim, cfg, seed):
    """pickUpPendingTasks under hdrf as vc_backfill_run computes it on the host (state rebuilt from allocate's
    operations, the tree evaluated on it) against the oracle's own live session after its allocate pass."""
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg, seed)
    hier, wts = H.random_tree(snap, np.random.default_rng(70 + seed))
    if seed % 2:
        H.swap_queue_order(snap)
    o = H.HdrfOracle(snap, hier, wts)
    dec, _, _ = o.allocate()
    want = o.backfill_pick_order()
    d, n, t, j, q, bt = snap.dims(), snap.nodes(), snap.tasks(), snap.jobs(), snap.queues(), snap.backfill_tasks()
    ops = np.ascontiguousarray(dec)
    out = np.zeros(max(snap.B, 1), np.int32)
    hd = snap.hdrf()
    got = shim.vhh_backfill_pick(C.byref(d), C.byref(snap.conf), C.byref(n), C.byref(t), C.byref(j), C.byref(q), C.byref(bt),
                                 snap.B, ops.ctypes.data_as(C.POINTER(abi.vc_decision)), len(ops), C.byref(hd),
                                 out.ctypes.data_as(_i32p))
    assert got == len(want) == snap.B
    assert list(out[:got]) == list(want)
