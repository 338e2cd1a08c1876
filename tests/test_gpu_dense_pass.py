"""The dense task x node pass (K1: vc_score_matrix / vc_dense_*) on every kernel path vc_dense_finish can take, against
the CPU oracle's score_matrix(), which scores every (task, node) pair with no grouping and no sharding. Mask, fp64
scores, best score and best node must be bit-identical.

vc_dense_finish picks its kernels from N, the shard start and the tunables: k_group_final + k_group_expand_bulk +
k_mask_expand_bulk for an even N and a shard start that is a multiple of 128, in node chunks of at most 8192 nodes;
otherwise the warp-store k_group_expand. Launches over more than 65 535 groups or work items go out in grid slices.
Every case asserts the precondition that puts it on its path, so a change of shapes cannot move it off unnoticed.

The last tests run parallel.sharded_dense_best in one thread per rank on one GPU, over a stand-in for torch.distributed
with NCCL's stream semantics, and stitch the ranks' matrices."""
import dataclasses
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SLICE = 65535  # grid-y limit: LAUNCH_Y_SLICED launches more groups / work items in slices


def _cfg(base, **changes):
    from volcano_b200.synth import CONFIGS
    return dataclasses.replace(CONFIGS[base], name=f"{base}-dense", **changes)


def _no_match_snapshot():
    """`small`, where the class of the first job selects two zones at once: no node carries both labels."""
    snap = _build(_cfg("small"))
    snap.c_selector[snap.t_klass[0], 0] = np.uint64(0b11)
    return snap


SNAPSHOTS = {
    "cfg2_t5k": lambda: _cfg("cfg2", n_tasks=5_000),
    "cfg2_fut_soft_t5k": lambda: _cfg("cfg2", n_tasks=5_000, releasing_frac=0.3, soft_taint_p=0.05),
    "n1": lambda: _cfg("tiny", n_nodes=1, n_tasks=64),
    "n64": lambda: _cfg("tiny"),
    "n65": lambda: _cfg("tiny", n_nodes=65),
    "n129": lambda: _cfg("tiny", n_nodes=129, n_tasks=600),
    "n700": lambda: _cfg("small"),
    "n701": lambda: _cfg("small", n_nodes=701),
    "n10001": lambda: _cfg("cfg2", n_nodes=10_001, n_tasks=3_000),
    "topo_n601": lambda: _cfg("small_topo", n_nodes=601),
    "n20000": lambda: _cfg("cfg2", n_nodes=20_000, n_tasks=3_000),
    "hetero_n200": lambda: _cfg("cfg2", n_nodes=200, n_tasks=80_000, hetero=400),
    "hetero_n201": lambda: _cfg("cfg2", n_nodes=201, n_tasks=80_000, hetero=400),
    "hetero_topo_n200": lambda: _cfg("small_topo", n_nodes=200, n_tasks=80_000, hetero=400, topology=(2, 3)),
    "t1": lambda: _cfg("small", n_tasks=1),
    "no_match": _no_match_snapshot,
    # almost full nodes, Releasing resources on every node: no task fits on Idle, many fit on FutureIdle
    "future_only": lambda: _cfg("small", utilisation=0.9999, min_util=0.999, releasing_frac=1.0),
    # sharded pass: terminating pods and PreferNoSchedule taints, so the all-reduced stats decide gradient and soft maximum
    "shard_n700": lambda: _cfg("small_fut_soft", n_nodes=700, n_tasks=3_000),
    "shard_n10000": lambda: _cfg("cfg2_fut_soft", n_tasks=2_000),
    "shard_n10001": lambda: _cfg("cfg2_fut_soft", n_nodes=10_001, n_tasks=2_000),
    "shard_n100": lambda: _cfg("small_fut_soft", n_nodes=100, n_tasks=500),
}


def _build(cfg):
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg)
    snap.synth_cfg = cfg
    return snap


def _make(name):
    from volcano_b200.synth import SynthConfig
    s = SNAPSHOTS[name]()
    return _build(s) if isinstance(s, SynthConfig) else s


def _nta(snap):
    return snap.hn_member is not None and "network-topology-aware" in snap.synth_cfg.plugins


@pytest.fixture(scope="module")
def gpu():
    from volcano_b200 import engine
    engine.init(0)
    return engine


@pytest.fixture(scope="module")
def oracle_of():
    """name -> (snapshot, oracle mask, score, best score, best node); the single-threaded oracle runs once per snapshot."""
    from oracle.pyoracle import OracleSession
    cache = {}

    def get(name):
        if name not in cache:
            snap = _make(name)
            o = OracleSession(snap)
            cache[name] = (snap, *o.score_matrix())
            o.close()
        return cache[name]

    return get


# ---- restatements of the host's grouping and launch geometry (preconditions only) ---------------------------------
def _groups(snap):
    """(group of every task, first task of every group): distinct (class, req_has | topology flag, resreq, k8s_req,
    k8s_nonzero_req) records, the key the library groups tasks by. The flag marks tasks of soft-mode topology jobs;
    the synthetic snapshots carry such jobs only together with the network-topology-aware plugin."""
    has = snap.t_req_has.astype(np.int64)
    soft = getattr(snap, "hn_job_soft", None)
    if soft is not None and soft.any():
        has = has | (soft[snap.t_job].astype(np.int64) << 30)

    def cols(a):
        return np.ascontiguousarray(np.asarray(a, np.float64).T).view(np.int64)

    key = np.concatenate([snap.t_klass.astype(np.int64)[:, None], has[:, None], cols(snap.t_resreq), cols(snap.t_k8s_req),
                          cols(snap.t_k8s_nonzero_req[:2])], axis=1)
    _, first, gid = np.unique(key, axis=0, return_index=True, return_inverse=True)
    return gid.ravel(), first


def _max_run(gid, rows):
    """Longest run of consecutive task ids inside one work item (`rows` tasks of one group, in task order)."""
    T = len(gid)
    order = np.argsort(gid, kind="stable")
    gs = gid[order]
    pos = np.arange(T) - np.searchsorted(gs, gs)
    item = gs.astype(np.int64) * (T + 1) + pos // rows
    brk = np.ones(T, bool)
    brk[1:] = (item[1:] != item[:-1]) | (order[1:] != order[:-1] + 1)
    starts = np.flatnonzero(brk)
    return int(np.diff(np.append(starts, T)).max())


def _geometry(snap, opts, begin=0, end=None):
    N = snap.N
    nloc = (N if end is None else end) - begin
    rows = opts.get("VC_EXPAND_ROWS", 0) or 16
    gid, _ = _groups(snap)
    sizes = np.bincount(gid)
    g = {"groups": len(sizes), "work": int((-(-sizes // rows)).sum()), "nloc": nloc,
         "path": "plain" if (N % 2 or begin % 128 or opts.get("VC_EXPAND_PLAIN", 0)) else "bulk"}
    if g["path"] == "bulk":
        max_chunk = max(128, opts["VC_EXPAND_CHUNK"] // 128 * 128) if opts.get("VC_EXPAND_CHUNK") else 8192
        nchunks = -(-nloc // max_chunk)
        chunk = (-(-nloc // nchunks) + 127) & ~127
        grid = -(-nloc // chunk)
        mw32 = (2 * ((N + 63) // 64) + 3) & ~3
        g.update(chunk=chunk, chunks=grid, last=nloc - (grid - 1) * chunk, pitch=mw32 * 4, rows=rows,
                 rows_cap=max(1, min(rows, 96 * 1024 // max(16, mw32 * 4))), max_run=_max_run(gid, rows))
    return g


# ---- checks ------------------------------------------------------------------------------------------------------
def _bits(mask, N):
    return np.unpackbits(np.ascontiguousarray(mask).view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)


def _assert_oracle(got, ref, what=""):
    mask, score, bs, bn = got
    omask, oscore, obs, obn = ref
    assert np.array_equal(mask, omask), f"{what}mask: {int((mask != omask).any(axis=1).sum())} rows differ"
    assert np.array_equal(score.view(np.int64), oscore.view(np.int64)), \
        f"{what}score: {int((score.view(np.int64) != oscore.view(np.int64)).sum())} cells differ"
    assert np.array_equal(bn, obn), f"{what}best node: {int((bn != obn).sum())} tasks differ"
    assert np.array_equal(bs.view(np.int64), obs.view(np.int64)), f"{what}best score: {int((bs != obs).sum())} tasks differ"


def _no_future(snap):
    return not snap.n_releasing.any() and not snap.n_pipelined.any()


def _invariants(snap, mask, score, bs, bn):
    """Properties of any dense-pass result, independent of the oracle."""
    N = snap.N
    gid, first = _groups(snap)
    rep = first[gid]
    assert np.array_equal(score.view(np.int64), score[rep].view(np.int64)), "rows of one group differ"
    assert np.array_equal(mask, mask[rep]), "mask rows of one group differ"
    if N % 64:
        assert not (mask[:, -1] >> np.uint64(N % 64)).any(), "mask bits past N"
    m = _bits(mask, N)
    assert not score[~m].any(), "score without a mask bit"
    if _no_future(snap):  # one candidate set: every feasible node; best = lowest index of the row maximum
        ms = np.where(m, score, -np.inf)
        top = ms.max(axis=1)
        empty = ~m.any(axis=1)
        want = np.where(empty, -1, np.argmax(ms == top[:, None], axis=1))
        assert np.array_equal(bn, want), f"best node is not the lowest-index maximum on {int((bn != want).sum())} rows"
        assert np.array_equal(bs, np.where(empty, 0.0, top))


def _pass(gpu, snap, opts):
    for k, v in opts.items():
        gpu.debug_option(k, v)
    try:
        e = gpu.Engine(snap)
        e.upload()
        out = e.score_matrix()
        e.close()
    finally:
        for k in opts:
            gpu.debug_option(k, 0)
    return out


# ---- one shard, every kernel path --------------------------------------------------------------------------------
CASES = [
    # several node chunks of k_group_expand_bulk, the last one short
    ("bulk_chunks", "cfg2_t5k", {}, {"path": "bulk", "chunks": 2, "chunk": 5120, "last": 4880}),
    ("bulk_chunk128", "cfg2_t5k", {"VC_EXPAND_CHUNK": 128}, {"path": "bulk", "chunks": 79, "last": 16}),
    ("bulk_chunk1000", "cfg2_t5k", {"VC_EXPAND_CHUNK": 1000}, {"path": "bulk", "chunk": 896, "last": 144}),
    ("bulk_chunks_fut_soft", "cfg2_fut_soft_t5k", {}, {"path": "bulk", "chunks": 2}),
    # k_group_expand: odd N (scalar stores), forced on even N (double2 stores), with the topology term
    ("plain_n1", "n1", {}, {"path": "plain"}),
    ("plain_n65", "n65", {}, {"path": "plain"}),
    ("plain_n129", "n129", {}, {"path": "plain"}),
    ("plain_n701", "n701", {}, {"path": "plain"}),
    ("plain_n10001", "n10001", {}, {"path": "plain"}),
    ("plain_forced_n64", "n64", {"VC_EXPAND_PLAIN": 1}, {"path": "plain"}),
    ("plain_forced_n700", "n700", {"VC_EXPAND_PLAIN": 1}, {"path": "plain"}),
    ("plain_forced_n10000", "cfg2_t5k", {"VC_EXPAND_PLAIN": 1}, {"path": "plain"}),
    ("plain_topo_n601", "topo_n601", {}, {"path": "plain"}),
    # k_mask_expand_bulk: runs of rows longer than the shared-memory row capacity are split
    ("mask_runs_split", "n20000", {"VC_EXPAND_ROWS": 100}, {"path": "bulk", "pitch": 2512, "rows_cap": 39}),
    ("mask_rows1", "n20000", {"VC_EXPAND_ROWS": 1}, {"path": "bulk", "rows_cap": 1}),
    # more than 65 535 groups (k_group_eval, k_group_best_partial, k_group_final, k_hn_scores) / work items
    ("sliced_groups_bulk", "hetero_n200", {}, {"path": "bulk"}),
    ("sliced_groups_plain", "hetero_n201", {}, {"path": "plain"}),
    ("sliced_groups_topo", "hetero_topo_n200", {}, {"path": "bulk"}),
    ("sliced_work_rows1", "hetero_n200", {"VC_EXPAND_ROWS": 1}, {"path": "bulk"}),
    # degenerate
    ("one_task", "t1", {}, {"path": "bulk"}),
    ("no_matching_node", "no_match", {}, {"path": "bulk"}),
    ("future_fit_only", "future_only", {}, {"path": "bulk"}),
]


def _assert_precondition(case, snap, opts, want, ref):
    g = _geometry(snap, opts)
    for k, v in want.items():
        assert g[k] == v, (k, g[k], v)
    omask, oscore, obs, obn = ref
    if case.startswith("plain_n") or case == "plain_topo_n601":
        assert snap.N % 2 == 1
    if case.startswith("plain_forced"):
        assert snap.N % 2 == 0
    if case == "plain_topo_n601":
        assert _nta(snap)
    if case.startswith("bulk_chunk"):
        assert snap.N > 8192 and g["chunks"] > 1 and g["last"] < g["chunk"]
    if case == "bulk_chunks_fut_soft":  # both categories and soft taints on either side of the chunk boundary
        for lo, hi in ((0, g["chunk"]), (g["chunk"], snap.N)):
            assert snap.n_releasing[:, lo:hi].any() and snap.n_taint_soft[0, lo:hi].any()
        assert (obn >= 0).sum() > 0
    if case == "mask_runs_split":
        assert g["rows_cap"] < 100 and g["max_run"] > g["rows_cap"], g
    if case.startswith("sliced_groups"):
        assert g["groups"] > SLICE, g
    if case == "sliced_groups_topo":
        assert _nta(snap)
    if case == "sliced_work_rows1":
        assert g["work"] > SLICE, g
    if case == "one_task":
        assert snap.T == 1 and obn[0] >= 0
    if case == "no_matching_node":
        empty = snap.t_klass == snap.t_klass[0]
        assert empty.any() and not omask[empty].any() and (obn[empty] == -1).all() and (obs[empty] == 0.0).all()
        assert (obn[~empty] >= 0).any()
    if case == "future_fit_only":  # no task fits on Idle cpu anywhere, but some fit on FutureIdle
        from volcano_b200.synth import D_CPU
        assert snap.n_idle[D_CPU].max() < snap.t_resreq[D_CPU].min()
        assert (obn >= 0).sum() > 100


@pytest.mark.parametrize("case,snap_name,opts,want", CASES, ids=[c[0] for c in CASES])
def test_dense_pass_vs_oracle(case, snap_name, opts, want, gpu, oracle_of):
    snap, *ref = oracle_of(snap_name)
    _assert_precondition(case, snap, opts, want, ref)
    got = _pass(gpu, snap, opts)
    _assert_oracle(got, ref)
    _invariants(snap, *got)


# ---- several passes on one engine --------------------------------------------------------------------------------
def test_second_pass_identical(gpu, oracle_of):
    """The matrix is zero-filled on the first pass only: the second pass must rewrite every cell it owns."""
    snap, *ref = oracle_of("n700")
    assert _geometry(snap, {})["path"] == "bulk"
    e = gpu.Engine(snap)
    e.upload()
    first = e.score_matrix()
    second = e.score_matrix()
    e.close()
    _assert_oracle(first, ref, "first pass: ")
    _assert_oracle(second, ref, "second pass: ")


def _move_nodes(snap, rng):
    """10 % of the nodes change: pods end on half of them, start on the other half; a few fill their pod slots
    (infeasible for every group), and the started pods make the larger groups infeasible elsewhere."""
    dirty = rng.choice(snap.N, size=snap.N // 10, replace=False).astype(np.int32)
    half = len(dirty) // 2
    unit = np.ones(snap.R)
    unit[snap.dim_names.index("nvidia.com/gpu")] = 1000.0
    for n in dirty[:half]:
        freed = np.floor(snap.n_used[:, n] / 2 / unit) * unit
        snap.n_used[:, n] -= freed
        snap.n_idle[:, n] += freed
    for n in dirty[half:]:
        taken = np.floor(snap.n_idle[:, n] * 0.9 / unit) * unit
        snap.n_used[:, n] += taken
        snap.n_idle[:, n] -= taken
    snap.n_pod_count[dirty] = snap.n_used[snap.pods_dim, dirty].astype(np.int32)
    snap.n_pod_count[dirty[:5]] = snap.n_max_tasks[dirty[:5]]
    kd = [snap.dim_names.index(k) for k in ("cpu", "memory", "nvidia.com/gpu")]
    for k, d in enumerate(kd):
        scale = 1000.0 if k == 2 else 1.0
        snap.n_k8s_requested[k, dirty] = snap.n_used[d, dirty] / scale
        snap.n_k8s_nonzero_requested[k, dirty] = snap.n_used[d, dirty] / scale
    return dirty


@pytest.mark.parametrize("plain", [0, 1], ids=["bulk", "plain"])
def test_pass_after_update_nodes(plain, gpu, oracle_of):
    """vc_snapshot_update_nodes between two passes on one engine: the second pass equals the oracle on the moved
    cluster, with no mask bit or score left from the first pass."""
    from oracle.pyoracle import OracleSession
    _, *ref0 = oracle_of("n700")
    snap = _make("n700")
    gpu.debug_option("VC_EXPAND_PLAIN", plain)
    try:
        e = gpu.Engine(snap)
        e.upload()
        _assert_oracle(e.score_matrix(), ref0, "before the move: ")
        dirty = _move_nodes(snap, np.random.default_rng(7))
        e.update_nodes(dirty, snap.n_idle[:, dirty], snap.n_used[:, dirty], snap.n_releasing[:, dirty],
                       snap.n_pipelined[:, dirty], snap.n_k8s_requested[:, dirty], snap.n_k8s_nonzero_requested[:, dirty],
                       snap.n_pod_count[dirty])
        got = e.score_matrix()
        e.close()
    finally:
        gpu.debug_option("VC_EXPAND_PLAIN", 0)
    o = OracleSession(snap)
    ref1 = o.score_matrix()
    o.close()
    # precondition: the move clears mask bits and changes scores of nodes that stay feasible
    m0, m1 = _bits(ref0[0], snap.N), _bits(ref1[0], snap.N)
    assert (m0 & ~m1).any()
    assert ((ref0[1] != ref1[1]) & m0 & m1).any()
    assert (~m1[:, dirty[:5]]).all()
    _assert_oracle(got, ref1, "after the move: ")
    _invariants(snap, *got)


def test_expand_plain_toggled_between_passes(gpu, oracle_of):
    snap, *ref = oracle_of("n700")
    assert snap.N % 2 == 0
    e = gpu.Engine(snap)
    e.upload()
    try:
        for plain in (0, 1, 0, 1):
            gpu.debug_option("VC_EXPAND_PLAIN", plain)
            _assert_oracle(e.score_matrix(), ref, f"VC_EXPAND_PLAIN={plain}: ")
    finally:
        gpu.debug_option("VC_EXPAND_PLAIN", 0)
        e.close()


def test_set_shard_sequence(gpu, oracle_of):
    """set_shard (0, N) -> (64, N) -> (0, N) on one engine. Without Releasing resources or soft taints a shard's
    stats cannot change a score, so the (64, N) shard holds the oracle's columns from 64 on, zeros before, and the
    lowest-index maximum of those columns as its best."""
    snap, *ref = oracle_of("n700")
    omask, oscore, obs, obn = ref
    N = snap.N
    assert _no_future(snap) and not snap.n_taint_soft.any()
    assert _geometry(snap, {}, 64, N)["path"] == "plain" and _geometry(snap, {})["path"] == "bulk"
    e = gpu.Engine(snap)
    e.upload()
    _assert_oracle(e.score_matrix(), ref, "(0, N): ")
    e.set_shard(64, N)
    mask, score, bs, bn = e.score_matrix()
    e.set_shard(0, N)
    again = e.score_matrix()
    with pytest.raises(gpu.VcError):
        e.set_shard(32, N)  # a shard with nodes begins at a multiple of 64
    e.set_shard(N, N)  # an empty one may begin anywhere: shard_bounds gives ranks past the last node [N, N)
    assert N % 64
    empty = e.score_matrix()
    e.close()
    assert not empty[0].any() and not empty[1].any() and not empty[2].any() and (empty[3] == -1).all()
    assert not mask[:, 0].any() and not score[:, :64].any()
    assert np.array_equal(mask[:, 1:], omask[:, 1:])
    assert np.array_equal(score[:, 64:].view(np.int64), oscore[:, 64:].view(np.int64))
    m = _bits(omask, N)[:, 64:]
    ms = np.where(m, oscore[:, 64:], -np.inf)
    top = ms.max(axis=1)
    empty = ~m.any(axis=1)
    assert np.array_equal(bn, np.where(empty, -1, 64 + np.argmax(ms == top[:, None], axis=1)))
    assert np.array_equal(bs, np.where(empty, 0.0, top))
    assert (bn != obn).any()  # some task's best lies in the first 64 nodes
    _assert_oracle(again, ref, "(0, N) again: ")


# ---- the node-sharded pass, one thread per rank on one GPU ---------------------------------------------------------
SLEEP_CYCLES = 20_000_000  # about 10 ms at the H100's 1.98 GHz boost clock


class _ThreadGroup:
    """Stand-in for torch.distributed across `world` threads on one GPU, with NCCL's stream semantics: a collective
    waits for every rank's input, is queued on the caller's current stream behind a few milliseconds of device sleep,
    and returns without a host synchronisation."""

    def __init__(self, world):
        import torch.distributed
        self.ReduceOp = torch.distributed.ReduceOp
        self.world = world
        self.barrier = threading.Barrier(world, timeout=120)
        self.lock = threading.Lock()
        self.rank_of = {}
        self.calls = [0] * world
        self.posted = {}  # call index -> [(input copy, event)] per rank; kept until the group is dropped

    def register(self, rank):
        self.rank_of[threading.get_ident()] = rank

    def get_world_size(self, group=None):
        return self.world

    def _exchange(self, tensor):
        import torch
        r = self.rank_of[threading.get_ident()]
        buf = tensor.clone()
        ev = torch.cuda.Event()
        ev.record()
        with self.lock:
            i = self.calls[r]
            self.calls[r] += 1
            self.posted.setdefault(i, [None] * self.world)[r] = (buf, ev)
        self.barrier.wait()
        cur = torch.cuda.current_stream()
        for _, e in self.posted[i]:
            cur.wait_event(e)
        torch.cuda._sleep(SLEEP_CYCLES)
        return [b for b, _ in self.posted[i]]

    def all_reduce(self, tensor, op=None, group=None, async_op=False):
        import torch
        assert op == self.ReduceOp.MAX and not async_op
        tensor.copy_(torch.stack(self._exchange(tensor)).amax(dim=0))

    def all_gather(self, tensor_list, tensor, group=None, async_op=False):
        assert not async_op
        for out, b in zip(tensor_list, self._exchange(tensor)):
            out.copy_(b)


def _load_kernels(gpu, snap, dev):
    """Launch every dense-pass kernel and the stand-in's torch kernels once before the ranks start: CUDA loads a kernel
    on its first launch and may synchronise the device to do so, which would hide a missing stream order."""
    import torch
    for plain in (0, 1):
        gpu.debug_option("VC_EXPAND_PLAIN", plain)
        try:
            e = gpu.Engine(snap)
            e.upload()
            e.score_matrix()
            e.close()
        finally:
            gpu.debug_option("VC_EXPAND_PLAIN", 0)
    x = torch.zeros(8, dtype=torch.int32, device=dev)
    x.copy_(torch.stack([x.clone(), x]).amax(dim=0))
    torch.cuda._sleep(1)
    torch.cuda.synchronize(dev)


def _fold(bests):
    """The canonical arg-max over shards: highest score, then lowest node; -1 / 0.0 where no shard has a candidate."""
    s = np.stack([b[0] for b in bests])
    n = np.stack([b[1] for b in bests]).astype(np.int64)
    s = np.where(n >= 0, s, -np.inf)
    top = s.max(axis=0)
    big = np.iinfo(np.int64).max
    node = np.where((n >= 0) & (s == top), n, big).min(axis=0)
    return np.where(node == big, 0.0, top), np.where(node == big, -1, node).astype(np.int32)


SHARDS = [
    # N, world, snapshot, what the shards reach
    (700, 2, "shard_n700", "bulk with a mask word offset in k_mask_expand_bulk; the stats reduction decides some bests"),
    (10_000, 2, "shard_n10000", "plain kernel on rank 1 (start 5056 = 64 mod 128)"),
    (10_001, 3, "shard_n10001", "odd N: plain kernel on every rank"),
    (100, 4, "shard_n100", "two empty shards (nloc == 0)"),
]


@pytest.mark.parametrize("N,world,snap_name,reach", SHARDS, ids=[f"n{s[0]}-w{s[1]}" for s in SHARDS])
def test_sharded_dense_pass_threads(N, world, snap_name, reach, gpu, oracle_of, monkeypatch):
    """parallel.sharded_dense_best, unmodified, in `world` threads with one Engine each: the stitched matrices and the
    folded best equal the oracle's full-axis pass."""
    import ctypes as C

    import torch

    from volcano_b200 import parallel
    snap, omask, oscore, obs, obn = oracle_of(snap_name)
    assert snap.N == N
    bounds = [parallel.shard_bounds(N, world, r) for r in range(world)]
    geo = [_geometry(snap, {}, b, e) for b, e in bounds]
    if N == 700:
        assert bounds[1][0] == 384 and geo[1]["path"] == "bulk"
    elif N == 10_000:
        assert bounds[1][0] % 128 == 64 and geo[0]["path"] == "bulk" and geo[1]["path"] == "plain"
    elif N == 10_001:
        assert all(g["path"] == "plain" for g in geo)
    else:
        assert sum(g["nloc"] == 0 for g in geo) == 2
    dev = torch.device("cuda", 0)
    _load_kernels(gpu, snap, dev)
    engines = [gpu.Engine(snap) for _ in range(world)]
    for e in engines:
        e.upload()
    fake = _ThreadGroup(world)
    monkeypatch.setattr(parallel, "dist", fake)
    results, errors = [None] * world, []

    def rank_main(r):
        try:
            torch.cuda.set_device(dev)
            with torch.cuda.stream(torch.cuda.Stream(device=dev)):
                fake.register(r)
                s, n = parallel.sharded_dense_best(engines[r], world, r, dev, materialize=True)
                results[r] = (s.cpu().numpy(), n.cpu().numpy())
        except BaseException as ex:  # noqa: BLE001 - re-raised in the main thread
            errors.append(ex)
            fake.barrier.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise errors[0]
        # each rank's matrix: its own columns and mask bits, zeros elsewhere; stitched, the oracle's full-axis matrix
        T, mw = snap.T, (N + 63) // 64
        bits = np.zeros((T, N), bool)
        score = np.zeros((T, N))
        for (b, e), eng in zip(bounds, engines):
            m = np.zeros((T, mw), np.uint64)
            sc = np.zeros((T, N))
            assert eng.L.vc_dense_fetch(eng.h, m.ctypes.data_as(C.POINTER(C.c_uint64)), sc.ctypes.data_as(C.POINTER(C.c_double)),
                                        None, None) == 0, eng.L.vc_last_error()
            mb = _bits(m, N)
            assert not mb[:, :b].any() and not mb[:, e:].any() and not sc[:, :b].any() and not sc[:, e:].any()
            if N % 64:
                assert not (m[:, -1] >> np.uint64(N % 64)).any()
            bits[:, b:e] = mb[:, b:e]
            score[:, b:e] = sc[:, b:e]
        assert np.array_equal(bits, _bits(omask, N)), f"mask: {int((bits != _bits(omask, N)).any(axis=1).sum())} rows differ"
        assert np.array_equal(score.view(np.int64), oscore.view(np.int64)), \
            f"score: {int((score.view(np.int64) != oscore.view(np.int64)).sum())} cells differ"
        for r, (bs, bn) in enumerate(results):
            assert np.array_equal(bn, obn), f"rank {r}: folded best node differs on {int((bn != obn).sum())} tasks"
            assert np.array_equal(bs.view(np.int64), obs.view(np.int64)), f"rank {r}: folded best score differs"
        # precondition of the first split: folding passes that score against each shard's local stats goes wrong
        if N == 700:
            local = []
            for (b, e), eng in zip(bounds, engines):
                eng.set_shard(b, e)
                _, _, bs, bn = eng.score_matrix(want_mask=False, want_score=False)
                local.append((bs, bn))
            assert (_fold(local)[1] != obn).any(), "the stats reduction changes no best on this snapshot"
    finally:
        for e in engines:
            e.close()
