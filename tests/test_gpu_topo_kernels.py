"""The topology-aware preemption kernels of vc_evict.cuh launched on their own (tools/kernels/evict_harness.cu, production
geometry): k_evict_dryrun against the exact Python restatement of SelectVictimsOnNode (tests/topo_kernels_common.py) and
k_evict_select against numpy.lexsort over the first numCandidates candidates in scan order from the offset."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import topo_kernels_common as K

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(HERE), "tools", "kernels", "_build", "evict_harness.so")


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB):
        pytest.fail(f"{LIB} is missing: build() compiles it")
    L = C.CDLL(LIB)
    L.eh_dryrun.argtypes = [C.POINTER(K.EhTopoArgs)]
    L.eh_select.argtypes = [C.POINTER(K.EhSelectArgs)]
    return L


@pytest.mark.parametrize("N,R,max_pods,seed", [(1, 2, 300, 0), (7, 16, 40, 1), (129, 9, 300, 2), (1000, 8, 300, 3),
                                               (1000, 16, 12, 4), (20_000, 4, 300, 8), (200_000, 16, 300, 9),
                                               (200_000, 3, 8, 7)])
def test_dryrun_matches_the_restatement(H, N, R, max_pods, seed):
    """Every node up to 1 000 nodes; beyond, 3 000 sampled nodes plus every node running more than 100 pods. Nodes run
    0-8 pods, a few up to `max_pods`; R up to 16 (both sides of the R <= 8 instance split of the other kernels); odd seeds
    use non-integer requests."""
    rng = np.random.default_rng(100 + seed)
    I = K.random_instance(rng, N, R, max_pods=max_pods, heavy=4, non_integer=seed % 2 == 1)
    if seed % 4 != 3:  # most cases without the quota gate, which rejects nearly every node at R = 16
        I.update(sim_state=1, q_exists=1, sim_alloc=0)
    a, out = K.to_args(I)
    assert H.eh_dryrun(C.byref(a)) == 0
    if N <= 1000:
        nodes = np.arange(N)
    else:
        pods = np.diff(I["rt_off"])
        nodes = np.union1d(rng.choice(N, 3000, replace=False), np.flatnonzero(pods > 100))
    hits = K.check_dry_run(I, out, nodes)
    assert N < 100 or seed % 4 == 3 or hits > 0


def _select_case(rng, N, levels):
    pred = (rng.random(N) < 0.8).astype(np.uint8)
    ok = (pred & (rng.random(N) < 0.5)).astype(np.uint8)
    keys = np.stack([rng.integers(0, levels, N) for _ in range(4)]).astype(np.int64)  # few values: ties at every level
    keys[0] -= 2 ** 40
    nv = np.where(ok == 1, 1, 0).astype(np.int32)
    rt_off = np.arange(N + 1, dtype=np.int32)
    victims = rng.integers(0, 10 ** 6, N).astype(np.int32)
    return pred, ok, keys, nv, rt_off, victims


COUNTS = {"0": (0, 0, 100), "1": (0, 1, 1), "10%": (10, 1, 10 ** 9), "100": (0, 100, 100), "all": (100, 1, 10 ** 9)}


@pytest.mark.parametrize("N", [1, 31, 1000, 4097, 100_000, 200_000])
@pytest.mark.parametrize("count", list(COUNTS))
def test_select_matches_lexsort(H, N, count):
    """Offsets from several seeds (wrap-around included), ties at every key level, numCandidates 0, 1, 10 %, 100, all."""
    pct, min_abs, max_abs = COUNTS[count]
    rng = np.random.default_rng(N * 7 + len(count))
    seq = 0
    for trial in range(4):
        pred, ok, keys, nv, rt_off, victims = _select_case(rng, N, [2, 3, 1, 5][trial])
        seed_k = int(rng.integers(0, 2 ** 63))
        words = np.zeros(K_SEQ(H) + 1, np.int32)
        seq += 1
        s = K.EhSelectArgs(N, N, *(x.ctypes.data_as(t) for x, t in ((pred, C.POINTER(C.c_uint8)), (ok, C.POINTER(C.c_uint8)),
                                                                       (nv, C.POINTER(C.c_int32)), (keys, C.POINTER(C.c_longlong)),
                                                                       (rt_off, C.POINTER(C.c_int32)), (victims, C.POINTER(C.c_int32)))),
                           seed_k, pct, min_abs, max_abs, seq, words.ctypes.data_as(C.POINTER(C.c_int32)))
        assert H.eh_select(C.byref(s)) == 0
        want, P = K.select(pred, ok, keys, seed_k, pct, min_abs, max_abs)
        assert words[K_SEQ(H)] == seq
        assert (words[0], words[2]) == (want, P), (trial, want, P, words[:4])
        if want >= 0:
            assert (words[1], words[3], words[4]) == (1, 0, victims[want])


def K_SEQ(H):
    H.eh_topo_seq_word.restype = C.c_int
    return H.eh_topo_seq_word()
