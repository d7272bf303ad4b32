"""The row-sharded embedding kernels at world sizes above one, on a single GPU.

dr_embed_fm_fwd_sharded / dr_embed_fm_bwd_sharded take every rank's shard as a raw base pointer (peer_bases) and never
ask which device it lives on, so W allocations on one device stand in for W ranks: global row r lives in allocation
r % W at local row r // W, laid out exactly as ShardedEmbedding lays out one rank's symmetric buffer
(shard_plan.p2p_layout).  At world 1 the owner is always 0 and the local row is the global row, so only W > 1 shows
whether a lookup reaches the right rank, row and first-order weight -- and only a W that is not a power of two runs
the modulo / divide form of that addressing.

Everything is checked against the float64 oracle of the unsharded table (tests/shard_oracle.py), and whatever does
not depend on summation order bit for bit against world 1 on the assembled table.  Every float of an allocation that
holds no live value -- the pad floats of a narrow row, the rows past a short rank's last one, the tail of the
first-order array, and guards on both sides large enough for any address formed from a valid global row -- holds a
sentinel that must survive.  The NCCL form of the exchange is emulated by slicing the padded segments by hand.
"""
import numpy as np
import pytest
import torch

import shard_oracle as O

pytestmark = pytest.mark.gpu

SENT = np.float32(-7777.25)
SENT_BITS = SENT.view(np.uint32)
PRE = 64          # floats of guard before each arena (keeps the arena 16-B aligned)
OUT_PAD = 256     # floats of guard on each side of an output

# ragged slot cardinalities (one single-row slot); the tiny table leaves ranks that own one row or none
TABLES = {"ragged": [301, 7, 1, 53, 997, 2, 129], "tiny": [5, 1, 2]}
WORLD_TABLES = [(w, "ragged") for w in (1, 2, 3, 4, 5, 6, 8)] + [(w, "tiny") for w in (3, 5, 6, 64)]
WT_IDS = [f"w{w}-{t}" for w, t in WORLD_TABLES]


def _lib():
    from deep_recommenders_b200 import _lib
    return _lib


def _st():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def streams():
    return [torch.cuda.Stream() for _ in range(64)]


class Guarded:
    """A float32 output of n elements between sentinel guards."""

    def __init__(self, n):
        self.n = n
        self.full = torch.full((n + 2 * OUT_PAD,), float(SENT), device="cuda")
        self.t = self.full[OUT_PAD:OUT_PAD + n]

    def get(self):
        f = self.full.cpu().numpy()
        assert (_bits(f[:OUT_PAD]) == SENT_BITS).all() and (_bits(f[OUT_PAD + self.n:]) == SENT_BITS).all(), \
            "store outside the output"
        return f[OUT_PAD:OUT_PAD + self.n]


class Arenas:
    """`world` shards of the global row space [sum(rows), D], one guarded allocation each, on the one GPU.

    layout: shard_plan.P2PLayout of one shard (default: the p2p DeepFM layout); lin None = no first-order weights."""

    def __init__(self, rows, D, world, table, lin, layout=None):
        from deep_recommenders_b200 import shard_plan
        self.rows, self.D, self.world = list(rows), D, world
        self.total = total = sum(rows)
        self.lay = lay = layout or shard_plan.p2p_layout(total, D, world)
        self.vdim, self.lin_offset, self.lin_in_row = lay.vdim, lay.lin_offset, lay.lin_in_row
        self.flags = 1 if lay.lin_in_row else 0
        self.has_lin = lin is not None
        self.nloc = [shard_plan.local_rows(total, g, world) for g in range(world)]
        # the guard behind each arena holds any row or first-order weight that a wrong owner / local split of a valid
        # global row can address (local < max(total, world)), so a misrouted access lands on a sentinel and is seen
        self.guard = (max(total, world) + 1) * lay.vdim + 64
        self.bufs, self.live = [], []
        for g in range(world):
            full = np.full(PRE + lay.numel + self.guard, SENT, np.float32)
            live = np.zeros(full.shape, bool)
            n = self.nloc[g]
            for arr, val in ((full, None), (live, True)):
                a = arr[PRE:PRE + lay.numel]
                rw = a[:lay.max_rows * lay.vdim].reshape(lay.max_rows, lay.vdim)
                rw[:n, :D] = table[g::world] if val is None else val
                if lin is not None:
                    if lay.lin_in_row:
                        rw[:n, D] = lin[g::world] if val is None else val
                    else:
                        a[lay.lin_offset:lay.lin_offset + n] = lin[g::world] if val is None else val
            self.bufs.append(torch.from_numpy(full).cuda())
            self.live.append(live)
        self.peer = torch.tensor([self.base(g) for g in range(world)], dtype=torch.int64, device="cuda")
        self.offs = torch.tensor(shard_plan.slot_offsets(self.rows), dtype=torch.int64, device="cuda")
        self.rows_t = torch.tensor(self.rows, dtype=torch.int64, device="cuda")

    def base(self, g):
        return self.bufs[g].data_ptr() + 4 * PRE

    def snapshot(self):
        return [b.cpu().numpy() for b in self.bufs]

    def gather(self):
        """Reassembled (table [total, D], lin [total] or None); asserts that every sentinel survived."""
        snap = self.snapshot()
        lay, D = self.lay, self.D
        table = np.empty((self.total, D), np.float32)
        lin = np.empty((self.total,), np.float32) if self.has_lin else None
        for g, (full, live) in enumerate(zip(snap, self.live)):
            assert (_bits(full[~live]) == SENT_BITS).all(), f"rank {g}: a dead float (pad / guard / spare row) changed"
            a, n = full[PRE:PRE + lay.numel], self.nloc[g]
            rw = a[:lay.max_rows * lay.vdim].reshape(lay.max_rows, lay.vdim)
            table[g::self.world] = rw[:n, :D]
            if lin is not None:
                lin[g::self.world] = rw[:n, D] if lay.lin_in_row else a[lay.lin_offset:lay.lin_offset + n]
        return table, lin


def make_table(rng, rows, D):
    total = sum(rows)
    return ((rng.standard_normal((total, D)) / np.sqrt(D)).astype(np.float32),
            (rng.standard_normal(total) * 0.1).astype(np.float32))


def zipf_ids(rng, n, rows, oov=0.08, a=1.3):
    """[n, S] Zipf ids (heavy duplicates spread over the rows by a random permutation) with OOV ids -1 and >= rows."""
    cols = []
    for r in rows:
        col = rng.permutation(r)[np.minimum(rng.zipf(a, n) - 1, r - 1)]
        bad = rng.random(n) < oov
        col[bad] = rng.choice(np.array([-1, r, r + 1, 1 << 30]), int(bad.sum()))
        cols.append(col)
    return np.stack(cols, 1).astype(np.int64)


def unique_ids(rng, n, rows):
    """[n, S] ids in which every global row is looked up at most once; the other lookups are OOV (-1 or rows[s])."""
    cols = []
    for r in rows:
        col = np.where(rng.random(n) < 0.5, -1, r).astype(np.int64)
        k = min(n, r)
        col[rng.choice(n, k, replace=False)] = rng.permutation(r)[:k]
        cols.append(col)
    return np.stack(cols, 1)


def fwd(ar, ids, bias, B, out_stack, out_sum, out_logit):
    L = _lib()
    L.check(L.load().dr_embed_fm_fwd_sharded(ar.peer.data_ptr(), ar.world, ar.offs.data_ptr(), ar.rows_t.data_ptr(),
                                             ids.data_ptr(), ids.element_size(), _ptr(bias), B, len(ar.rows), ar.D,
                                             ar.vdim, ar.flags, ar.lin_offset, _ptr(out_stack), _ptr(out_sum),
                                             _ptr(out_logit), _st()), "dr_embed_fm_fwd_sharded")


def bwd(ar, ids, stack, sum_e, g_logit, g_stack, g_bias, scale, B):
    L = _lib()
    L.check(L.load().dr_embed_fm_bwd_sharded(ar.peer.data_ptr(), ar.world, ar.offs.data_ptr(), ar.rows_t.data_ptr(),
                                             ids.data_ptr(), ids.element_size(), _ptr(stack), _ptr(sum_e),
                                             _ptr(g_logit), _ptr(g_stack), B, len(ar.rows), ar.D, ar.vdim, ar.flags,
                                             ar.lin_offset, _ptr(g_bias), scale, _st()), "dr_embed_fm_bwd_sharded")


def run_fwd(ar, ids_t, B):
    S, D = len(ar.rows), ar.D
    outs = Guarded(B * S * D), Guarded(B * D), Guarded(B)
    bias = torch.tensor([0.3], device="cuda")
    fwd(ar, ids_t, bias, B, *(o.t for o in outs))
    torch.cuda.synchronize()
    return [o.get().copy() for o in outs]


def check_fwd(outs, ref):
    stack, s, logit = outs
    ref_stack, sum64, sum_abs, logit64, lscale = ref
    assert np.array_equal(_bits(stack), _bits(ref_stack.reshape(-1))), "gathered rows are not a copy of the table"
    err = np.abs(s.astype(np.float64) - sum64.reshape(-1))
    assert (err <= 1e-5 * sum_abs.reshape(-1) + 1e-7).all(), f"sum_e: max err {err.max()}"
    err = np.abs(logit.astype(np.float64) - logit64)
    tol = 1e-5 * lscale + 1e-6
    assert (err <= tol).all(), f"logit: max err {err.max()} at {np.argmax(err / tol)}"


# ---- forward --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("id_dtype", [np.int64, np.int32], ids=["i64", "i32"])
@pytest.mark.parametrize("D", [16, 12, 32, 128])
@pytest.mark.parametrize("world,tname", WORLD_TABLES, ids=WT_IDS)
def test_forward_matches_oracle_and_world1(world, tname, D, id_dtype):
    """stack / sum_e / logit at world W: the oracle, and bit for bit world 1 on the assembled arena (only the
    addressing differs).  In-row weights also under the LINX lane mapping (knob embed_fwd_linx_shard)."""
    L = _lib()
    rows, S, B = TABLES[tname], len(TABLES[tname]), 203        # B: no multiple of any lane-group count
    rng = np.random.default_rng(world * 1000 + D)
    table, lin = make_table(rng, rows, D)
    ids = zipf_ids(rng, B, rows).astype(id_dtype)
    ids_t = _dev(ids)
    ar, ar1 = Arenas(rows, D, world, table, lin), Arenas(rows, D, 1, table, lin)
    before, before1 = ar.snapshot(), ar1.snapshot()
    ref = O.fm_forward(table, lin, 0.3, rows, ids)
    first = None
    for linx in ([0, 1] if ar.lin_in_row and world > 1 else [0]):
        L.tune("embed_fwd_linx_shard", linx)
        try:
            outs, outs1 = run_fwd(ar, ids_t, B), run_fwd(ar1, ids_t, B)
        finally:
            L.tune("embed_fwd_linx_shard", 0)
        check_fwd(outs, ref)
        for name, a, b in zip(("stack", "sum_e", "logit"), outs, outs1):
            assert np.array_equal(_bits(a), _bits(b)), f"linx={linx}: {name} at world {world} != world 1"
        if first is None:
            first = outs
        for name, a, b in zip(("stack", "sum_e", "logit"), outs, first):
            assert np.array_equal(_bits(a), _bits(b)), f"{name}: the LINX mapping changed the numbers"
    for b0, b1 in zip(before + before1, ar.snapshot() + ar1.snapshot()):
        assert np.array_equal(_bits(b0), _bits(b1)), "the forward wrote into an arena"


# ---- backward: one global step, W ranks updating the shared arenas ---------------------------------------------------
GRADS = ["logit", "stack", "both"]


def grads_for(rng, kind, N, S, D):
    g_logit = rng.standard_normal(N).astype(np.float32) if kind in ("logit", "both") else None
    g_stack = rng.standard_normal((N, S, D)).astype(np.float32) if kind in ("stack", "both") else None
    return g_logit, g_stack


def step_ranks(ar, world, B, ids_t, stack_t, sum_t, gl_t, gs_t, g_bias, scale, streams=None):
    """Rank g runs the backward on its slice [g B, (g+1) B) with scale -lr / W, as ShardedDeepFMTrainStep does;
    sequentially on the current stream, or all at once on one stream per rank."""
    main = torch.cuda.current_stream()
    sl = lambda t, g: None if t is None else t[g * B:(g + 1) * B]
    for g in range(world):
        if streams is None:
            bwd(ar, sl(ids_t, g), sl(stack_t, g), sl(sum_t, g), sl(gl_t, g), sl(gs_t, g), g_bias, scale, B)
        else:
            streams[g].wait_stream(main)
            with torch.cuda.stream(streams[g]):
                bwd(ar, sl(ids_t, g), sl(stack_t, g), sl(sum_t, g), sl(gl_t, g), sl(gs_t, g), g_bias, scale, B)
    if streams is not None:
        for g in range(world):
            main.wait_stream(streams[g])
    torch.cuda.synchronize()


def check_update(ar, table, lin, rows, ids, g_logit, g_stack, scale, g_bias):
    got_t, got_l = ar.gather()
    want_t, want_l, bound_t, bound_l, touched = O.sgd_step(table, lin, rows, ids, g_logit, g_stack, scale)
    err = np.abs(got_t - want_t)
    assert (err <= bound_t).all(), f"table: max err {err.max()} (row {np.argmax(err.max(1))})"
    err = np.abs(got_l - want_l)
    assert (err <= bound_l).all(), f"first-order weights: max err {err.max()} (row {np.argmax(err)})"
    assert np.array_equal(_bits(got_t[~touched]), _bits(table[~touched])), "a row no lookup touched changed"
    assert np.array_equal(_bits(got_l[~touched]), _bits(lin[~touched])), "a weight no lookup touched changed"
    if g_logit is None:
        assert np.array_equal(_bits(got_l), _bits(lin)), "first-order weights moved without g_logit"
        assert float(g_bias) == 0.0
    else:
        gl = np.asarray(g_logit, np.float64)
        assert abs(float(g_bias) - scale * gl.sum()) <= 1e-5 * abs(scale) * np.abs(gl).sum() + 1e-7
    return got_t, got_l


def _saved(table, lin, rows, ids):
    """What the forward saved for the backward: the exact fp32 gather [N, S, D] and its fp32 sum over the slots."""
    from oracle import reference_np as R
    tables, _ = O.split(table, lin, rows)
    stack_t = _dev(R.stack_embeddings(tables, ids))
    return stack_t, stack_t.sum(1).contiguous()


@pytest.mark.parametrize("grads", GRADS)
@pytest.mark.parametrize("D", [16, 12, 32, 128])
@pytest.mark.parametrize("world,tname", WORLD_TABLES, ids=WT_IDS)
def test_backward_sequential_bit_identical_to_world1(world, tname, D, grads):
    """Every global row hit at most once: one vector atomic per row, so the reassembled table and first-order weights
    at world W are bit-identical to world 1 running the same slices (int32 ids here, int64 in the concurrent form)."""
    rows, S, B = TABLES[tname], len(TABLES[tname]), 45
    rng = np.random.default_rng(world * 7 + D)
    table, lin = make_table(rng, rows, D)
    ids = unique_ids(rng, world * B, rows).astype(np.int32)
    g_logit, g_stack = grads_for(rng, grads, world * B, S, D)
    ids_t, gl_t, gs_t = _dev(ids), _dev(g_logit), _dev(g_stack)
    stack_t, sum_t = _saved(table, lin, rows, ids)
    scale = -0.5 / world
    ar, ar1 = Arenas(rows, D, world, table, lin), Arenas(rows, D, 1, table, lin)
    gb, gb1 = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    step_ranks(ar, world, B, ids_t, stack_t, sum_t, gl_t, gs_t, gb, scale)
    step_ranks(ar1, world, B, ids_t, stack_t, sum_t, gl_t, gs_t, gb1, scale)
    got_t, got_l = check_update(ar, table, lin, rows, ids, g_logit, g_stack, scale, gb)
    one_t, one_l = check_update(ar1, table, lin, rows, ids, g_logit, g_stack, scale, gb1)
    assert np.array_equal(_bits(got_t), _bits(one_t)), f"table at world {world} != world 1"
    assert np.array_equal(_bits(got_l), _bits(one_l)), f"first-order weights at world {world} != world 1"


@pytest.mark.parametrize("grads", GRADS)
@pytest.mark.parametrize("D", [16, 12, 32, 128])
@pytest.mark.parametrize("world,tname", WORLD_TABLES, ids=WT_IDS)
def test_backward_concurrent_matches_oracle(world, tname, D, grads, streams):
    """Zipf-heavy ids, the W slices launched on W streams at once: atomics of different ranks land on the same owner
    rows in any order; table, first-order weights and the bias gradient against the float64 row-sparse SGD step."""
    rows, S, B = TABLES[tname], len(TABLES[tname]), 45
    rng = np.random.default_rng(world * 11 + D)
    table, lin = make_table(rng, rows, D)
    ids = zipf_ids(rng, world * B, rows, a=1.1)
    g_logit, g_stack = grads_for(rng, grads, world * B, S, D)
    ids_t, gl_t, gs_t = _dev(ids), _dev(g_logit), _dev(g_stack)
    stack_t, sum_t = _saved(table, lin, rows, ids)
    scale = -0.5 / world
    ar = Arenas(rows, D, world, table, lin)
    gb = torch.zeros(1, device="cuda")
    step_ranks(ar, world, B, ids_t, stack_t, sum_t, gl_t, gs_t, gb, scale, streams)
    check_update(ar, table, lin, rows, ids, g_logit, g_stack, scale, gb)


# ---- two-tower form: S = 1, rows of D floats, no first-order term, g_stack only ------------------------------------
TT_TABLES = {"ragged": (37, 53), "tiny": (3, 5)}
TT_WORLDS = [(w, "ragged") for w in (1, 2, 3, 4, 5, 6, 8)] + [(w, "tiny") for w in (3, 5, 6, 64)]


@pytest.mark.parametrize("D", [16, 64])
@pytest.mark.parametrize("world,tname", TT_WORLDS, ids=[f"w{w}-{t}" for w, t in TT_WORLDS])
def test_two_tower_gather_and_update(world, tname, D, streams):
    """ShardedTwoTowerTrainStep._gather / _update: users then items in one row space, every rank on its own stream."""
    from deep_recommenders_b200 import shard_plan
    L = _lib()
    lib = L.load()
    U, I = TT_TABLES[tname]
    b, lr = 29, 0.05
    rng = np.random.default_rng(world * 13 + D)
    table, _ = make_table(rng, [U, I], D)
    max_rows = shard_plan.local_rows(U + I, 0, world)
    ar = Arenas([U, I], D, world, table, None, shard_plan.P2PLayout(max_rows, D, False, 0, max_rows * D))
    uid, iid = zipf_ids(rng, world * b, [U]), zipf_ids(rng, world * b, [I])
    i64 = dict(dtype=torch.int64, device="cuda")
    tower = [(torch.tensor([0], **i64), torch.tensor([U], **i64), _dev(uid), 0, U),
             (torch.tensor([U], **i64), torch.tensor([I], **i64), _dev(iid), U, I)]
    for off, rws, ids_t, o, r in tower:
        for g in range(world):
            out = Guarded(b * D)
            L.check(lib.dr_embed_fm_fwd_sharded(ar.peer.data_ptr(), world, off.data_ptr(), rws.data_ptr(),
                                                ids_t[g * b:].data_ptr(), 8, None, b, 1, D, D, 0, 0, out.t.data_ptr(),
                                                None, None, _st()), "dr_embed_fm_fwd_sharded")
            got = out.get().reshape(b, D)
            ids = ids_t[g * b:(g + 1) * b, 0].cpu().numpy()
            ok = (ids >= 0) & (ids < r)
            want = np.zeros((b, D), np.float32)
            want[ok] = table[o + ids[ok]]
            assert np.array_equal(_bits(got), _bits(want)), f"rank {g}: gathered rows"
    grads = [rng.standard_normal((world * b, D)).astype(np.float32) for _ in tower]
    grads_t = [_dev(gr) for gr in grads]
    main = torch.cuda.current_stream()
    for g in range(world):
        streams[g].wait_stream(main)
        with torch.cuda.stream(streams[g]):
            for (off, rws, ids_t, _, _), gr in zip(tower, grads_t):
                L.check(lib.dr_embed_fm_bwd_sharded(ar.peer.data_ptr(), world, off.data_ptr(), rws.data_ptr(),
                                                    ids_t[g * b:].data_ptr(), 8, None, None, None, gr[g * b:].data_ptr(),
                                                    b, 1, D, D, 0, 0, None, -lr, _st()), "dr_embed_fm_bwd_sharded")
    for g in range(world):
        main.wait_stream(streams[g])
    torch.cuda.synchronize()
    want = torch.from_numpy(table).double()
    scale = torch.from_numpy(np.abs(table)).double()
    touched = np.zeros(U + I, bool)
    for (_, _, ids_t, o, r), gr in zip(tower, grads):
        ids = ids_t[:, 0].cpu().numpy()
        ok = (ids >= 0) & (ids < r)
        rows_ok = torch.from_numpy(o + ids[ok])
        want.index_add_(0, rows_ok, -lr * torch.from_numpy(gr[ok]).double())
        scale.index_add_(0, rows_ok, lr * torch.from_numpy(np.abs(gr[ok])).double())
        touched[o + ids[ok]] = True
    got, _ = ar.gather()
    err = np.abs(got - want.numpy())
    assert (err <= 1e-5 * scale.numpy() + 1e-7).all(), f"max err {err.max()}"
    assert np.array_equal(_bits(got[~touched]), _bits(table[~touched])), "a row no lookup touched changed"


# ---- the NCCL exchange, emulated in one process ---------------------------------------------------------------------
def bucket(ids_t, n, S, offs, rows_t, G, cap):
    L = _lib()
    counts = torch.zeros(G, dtype=torch.int64, device="cuda")
    send = torch.empty(G * cap, dtype=torch.int64, device="cuda")
    inv = torch.empty(n, dtype=torch.int32, device="cuda")
    ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(L.load().dr_shard_bucket_ids(ids_t.data_ptr(), ids_t.element_size(), n, S, offs.data_ptr(),
                                         rows_t.data_ptr(), G, cap, counts.data_ptr(), send.data_ptr(), inv.data_ptr(),
                                         ovf.data_ptr(), _st()), "dr_shard_bucket_ids")
    return counts, send, inv, ovf


@pytest.mark.parametrize("id_dtype", [np.int64, np.int32], ids=["i64", "i32"])
@pytest.mark.parametrize("G", [2, 3, 5, 8])
def test_bucket_ids_matches_numpy_twin(G, id_dtype):
    from deep_recommenders_b200 import shard_plan
    from oracle import shard_np
    rows = TABLES["ragged"]
    S, B = len(rows), 333
    ids = zipf_ids(np.random.default_rng(G), B, rows).astype(id_dtype)
    offs = shard_plan.slot_offsets(rows)
    cap = shard_plan.capacity(B * S, G, slack=1.0, floor=16)
    offs_t, rows_t = _dev(np.array(offs, np.int64)), _dev(np.array(rows, np.int64))
    counts, send, inv, ovf = bucket(_dev(ids), B * S, S, offs_t, rows_t, G, cap)
    rsend, rinv, rcounts, rovf = shard_np.bucket_ids(ids, offs, rows, G, cap)
    assert int(ovf) == int(rovf) == 0
    assert np.array_equal(counts.cpu().numpy(), rcounts)
    send_np, inv_np = send.cpu().numpy(), inv.cpu().numpy()
    for g in range(G):      # order inside a segment is unspecified: the multiset per segment
        assert np.array_equal(np.sort(send_np[g * cap:(g + 1) * cap]), np.sort(rsend[g * cap:(g + 1) * cap]))
    lv = rinv >= 0
    assert np.array_equal(inv_np >= 0, lv)
    assert np.array_equal(send_np[inv_np[lv]], rsend[rinv[lv]])
    assert np.array_equal(inv_np[lv] // cap, rinv[lv] // cap)
    assert len(np.unique(inv_np[lv])) == int(lv.sum())


NCCL_CASES = [(2, "ragged"), (3, "ragged"), (5, "ragged"), (8, "ragged"), (3, "tiny"), (5, "tiny")]


@pytest.mark.parametrize("D", [16, 12, 32])
@pytest.mark.parametrize("G,tname", NCCL_CASES, ids=[f"w{w}-{t}" for w, t in NCCL_CASES])
def test_nccl_exchange_emulated(G, tname, D):
    """exchange='nccl' of ShardedDeepFMTrainStep with the all-to-alls done by slicing: bucket, owner gather of fused
    rows [emb | w | pad], identity-table forward on the receive buffer, gradient pack, owner scatter with -lr / G.
    The forward equals the p2p forward; the update equals the float64 row-sparse SGD step."""
    from deep_recommenders_b200 import shard_plan
    L = _lib()
    lib = L.load()
    rows, S, B = TABLES[tname], len(TABLES[tname]), 45
    V, lr = D + 4, 0.5
    rng = np.random.default_rng(G * 17 + D)
    table, lin = make_table(rng, rows, D)
    ids = zipf_ids(rng, G * B, rows, a=1.1)
    g_logit, g_stack = grads_for(rng, "both", G * B, S, D)
    ids_t, gl_t, gs_t = _dev(ids), _dev(g_logit), _dev(g_stack)
    p2p = Arenas(rows, D, G, table, lin)
    mx = shard_plan.local_rows(sum(rows), 0, G)
    own = Arenas(rows, D, G, table, lin, shard_plan.P2PLayout(mx, V, True, 0, mx * V))   # pad floats = sentinel
    cap = shard_plan.capacity(B * S, G)
    bias = torch.tensor([0.3], device="cuda")
    f32 = dict(dtype=torch.float32, device="cuda")
    # requesters: bucket their lookups by owner
    plans = [bucket(ids_t[r * B:(r + 1) * B], B * S, S, own.offs, own.rows_t, G, cap) for r in range(G)]
    seg = lambda t, k: t[k * cap:(k + 1) * cap]
    recv_ids = [torch.cat([seg(plans[r][1], o) for r in range(G)]) for o in range(G)]            # a2a ids
    vec_send = [torch.empty((G * cap, V), **f32) for _ in range(G)]
    for o in range(G):
        L.check(lib.dr_gather_fwd(own.base(o), own.nloc[o], recv_ids[o].data_ptr(), 8, G * cap, V,
                                  vec_send[o].data_ptr(), _st()), "dr_gather_fwd")
    vec_recv = [torch.cat([seg(vec_send[o], r) for o in range(G)]) for r in range(G)]             # a2a vectors
    grad_send = [torch.zeros((G * cap, V), **f32) for _ in range(G)]
    i64 = dict(dtype=torch.int64, device="cuda")
    trows = torch.full((S,), G * cap, **i64)
    keep = []
    for r in range(G):
        _, _, inv, ovf = plans[r]
        assert int(ovf) == 0
        sl = slice(r * B, (r + 1) * B)
        out = Guarded(B * S * D), Guarded(B * D), Guarded(B)
        tp = torch.full((S,), vec_recv[r].data_ptr(), **i64)
        lp = torch.full((S,), vec_recv[r].data_ptr() + 4 * D, **i64)
        L.check(lib.dr_embed_fm_fwd(tp.data_ptr(), lp.data_ptr(), trows.data_ptr(), inv.data_ptr(), 4, bias.data_ptr(),
                                    B, S, D, V, V, 1, *(o.t.data_ptr() for o in out), _st()), "dr_embed_fm_fwd")
        got = [o.get() for o in out]
        want = run_fwd(p2p, ids_t[sl], B)
        check_fwd(got, O.fm_forward(table, lin, 0.3, rows, ids[sl]))
        names = ("stack", "sum_e", "logit") if D + 1 <= 32 else ("stack", "sum_e")   # wide p2p rows sum the
        for name, a, b in zip(names, got, want):                                       # weights in another order
            assert np.array_equal(_bits(a), _bits(b)), f"rank {r}: {name} of the nccl path != p2p"
        gb = torch.zeros(1, **f32)
        gtp = torch.full((S,), grad_send[r].data_ptr(), **i64)
        glp = torch.full((S,), grad_send[r].data_ptr() + 4 * D, **i64)
        stack, sum_e = out[0].t, out[1].t
        L.check(lib.dr_embed_fm_bwd(inv.data_ptr(), 4, trows.data_ptr(), stack.data_ptr(), sum_e.data_ptr(),
                                    gl_t[sl].data_ptr(), gs_t[sl].data_ptr(), B, S, D, V, V, 1, gtp.data_ptr(),
                                    glp.data_ptr(), gb.data_ptr(), 1.0, _st()), "dr_embed_fm_bwd(pack)")
        gl = g_logit[sl].astype(np.float64)
        assert abs(float(gb) - gl.sum()) <= 1e-5 * np.abs(gl).sum() + 1e-7
        keep.append((out, tp, lp, gtp, glp))
    grad_recv = [torch.cat([seg(grad_send[r], o) for r in range(G)]) for o in range(G)]           # a2a gradients
    for o in range(G):
        L.check(lib.dr_scatter_add(own.base(o), own.nloc[o], recv_ids[o].data_ptr(), 8, G * cap, V,
                                   grad_recv[o].data_ptr(), -lr / G, _st()), "dr_scatter_add")
    torch.cuda.synchronize()
    got_t, got_l = own.gather()
    want_t, want_l, bound_t, bound_l, touched = O.sgd_step(table, lin, rows, ids, g_logit, g_stack, -lr / G)
    assert (np.abs(got_t - want_t) <= bound_t).all(), np.abs(got_t - want_t).max()
    assert (np.abs(got_l - want_l) <= bound_l).all(), np.abs(got_l - want_l).max()
    assert np.array_equal(_bits(got_t[~touched]), _bits(table[~touched]))
    assert np.array_equal(_bits(got_l[~touched]), _bits(lin[~touched]))


# ---- dr_permute_rows / dr_unpermute_rows ----------------------------------------------------------------------------
@pytest.mark.parametrize("n,D", [(1, 4), (77, 12), (1000, 16), (333, 128)])
def test_permute_and_unpermute_rows(n, D):
    """out[i] = in[perm[i]] and out[perm[i]] = in[i]; a negative perm entry is skipped (that row is not written)."""
    L = _lib()
    lib = L.load()
    rng = np.random.default_rng(n + D)
    x = rng.standard_normal((n, D)).astype(np.float32)
    xt = _dev(x)
    skip = rng.random(n) < 0.25
    for un in (False, True):
        perm = (rng.permutation(n) if un else rng.integers(0, n, n)).astype(np.int32)   # a gather may repeat rows
        perm[skip] = -1 - rng.integers(0, 3, int(skip.sum()))
        want = np.full((n, D), SENT, np.float32)
        ok = perm >= 0
        if un:
            want[perm[ok]] = x[ok]
        else:
            want[ok] = x[perm[ok]]
        out, perm_t = Guarded(n * D), _dev(perm)
        fn = lib.dr_unpermute_rows if un else lib.dr_permute_rows
        L.check(fn(xt.data_ptr(), perm_t.data_ptr(), n, D, out.t.data_ptr(), _st()), "dr_(un)permute_rows")
        assert np.array_equal(_bits(out.get()), _bits(want.reshape(-1))), f"unpermute={un}"
    L.check(lib.dr_permute_rows(xt.data_ptr(), perm_t.data_ptr(), 0, D, out.t.data_ptr(), _st()), "dr_permute_rows(n=0)")
    assert np.array_equal(_bits(out.get()), _bits(want.reshape(-1))), "n = 0 wrote"
