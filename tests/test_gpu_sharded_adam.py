"""tf.keras-equal Adam on the row-sharded DeepFM tables (dr_shard_adam_mark / _prepare / _apply, optimizer="adam_rows_tf"
of ShardedDeepFMTrainStep).

Emulated worlds: as in test_gpu_sharded_emulated.py, W guarded allocations on one GPU stand in for W ranks (the kernels
take every rank's shard, gradient arena and touch array as raw base pointers).  Each step runs, rank by rank, what the
trainer runs: mark -> prepare (list + replay) -> sharded forward -> sharded backward of synthetic g_logit / g_stack
into the gradient arenas with scale 1/W -> apply; after the last step every rank flushes.  The tables, first-order
weights, m and v are held to a float64 model of dense Adam on the unsharded table and global batch, and -- with ids that
hit every row at most once per step, so no atomic order is involved -- bit for bit to world 1 running the same slices.

Real trainer at world 1 (p2p and nccl exchanges): against DeepFMTrainStep(optimizer="adam_rows_tf") from the same
weights; graph replay against eager; capture() side-effect free; save -> load -> continue against an uninterrupted run.
"""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_gpu_sharded_emulated import TABLES, Arenas, _bits, _dev, _lib, _st, bwd, fwd, make_table, zipf_ids

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LR, B1, B2, EPS = 0.01, 0.9, 0.999, 1e-7
STEPS = 6
HIST = 2            # small rate ring: rows that sat out more than 2 steps take the recomputed rate
WORLD_TABLES = [(w, "ragged") for w in (1, 2, 3, 5, 8)] + [(w, "tiny") for w in (3, 64)]
WT_IDS = [f"w{w}-{t}" for w, t in WORLD_TABLES]


class Ranks:
    """Per-rank Adam state of an emulated world: gradient arenas (guarded like the shards), touch arrays, row lists,
    counts and state blocks, with one clock (every rank advances an identical one)."""

    def __init__(self, ar: Arenas, hist):
        from deep_recommenders_b200 import ops
        lib = _lib().load()
        self.ar = ar
        zt, zl = np.zeros((ar.total, ar.D), np.float32), np.zeros(ar.total, np.float32)
        self.grad = Arenas(ar.rows, ar.D, ar.world, zt, zl, ar.lay)
        i32 = dict(dtype=torch.int32, device="cuda")
        self.touch = [torch.zeros(max(1, ar.lay.max_rows), **i32) for _ in range(ar.world)]
        self.touch_peer = torch.tensor([t.data_ptr() for t in self.touch], dtype=torch.int64, device="cuda")
        self.list = [torch.zeros(max(1, n), **i32) for n in ar.nloc]
        self.count = [torch.zeros(1, **i32) for _ in ar.nloc]
        self.SS = lib.dr_embed_adam_state_stride(ar.D)
        self.state = [torch.zeros((max(1, n), self.SS), device="cuda") for n in ar.nloc]
        self.clock = ops.AdamClock(LR, B1, B2, EPS, device="cuda", history=hist)

    def mark(self, ids_t, B):
        L, ck = _lib(), self.clock
        L.check(L.load().dr_shard_adam_mark(ids_t.data_ptr(), ids_t.element_size(), B * len(self.ar.rows),
                                            len(self.ar.rows), self.ar.offs.data_ptr(), self.ar.rows_t.data_ptr(),
                                            self.ar.world, self.touch_peer.data_ptr(), ck.step.data_ptr(), _st()),
                "dr_shard_adam_mark")

    def prepare(self, g):
        L, ar, ck = _lib(), self.ar, self.clock
        L.check(L.load().dr_shard_adam_prepare(self.touch[g].data_ptr(), ar.nloc[g], self.list[g].data_ptr(),
                                               self.count[g].data_ptr(), ar.D, ar.vdim, ar.lin_offset, ar.flags,
                                               ar.base(g), self.state[g].data_ptr(), ck.step.data_ptr(),
                                               ck.lr_hist.data_ptr(), ck.lr_hist.numel(), LR, B1, B2, EPS, _st()),
                "dr_shard_adam_prepare")

    def apply(self, g):
        L, ar, ck = _lib(), self.ar, self.clock
        L.check(L.load().dr_shard_adam_apply(self.list[g].data_ptr(), self.count[g].data_ptr(), ar.nloc[g], ar.D,
                                             ar.vdim, ar.lin_offset, ar.flags, ar.base(g), self.grad.base(g),
                                             self.state[g].data_ptr(), ck.step.data_ptr(), ck.lr_t.data_ptr(), B1, B2,
                                             EPS, _st()), "dr_shard_adam_apply")

    def flush(self, g):
        L, ar, ck = _lib(), self.ar, self.clock
        i64 = dict(dtype=torch.int64, device="cuda")
        rows, offs = torch.tensor([ar.nloc[g]], **i64), torch.zeros(1, **i64)
        tp, lp = torch.tensor([ar.base(g)], **i64), torch.tensor([ar.base(g) + 4 * ar.lin_offset], **i64)
        L.check(L.load().dr_embed_adam_flush(rows.data_ptr(), offs.data_ptr(), 1, ar.D, ar.nloc[g], ar.vdim, 1,
                                             ar.flags, tp.data_ptr(), lp.data_ptr(), self.state[g].data_ptr(),
                                             ck.step.data_ptr(), ck.lr_hist.data_ptr(), ck.lr_hist.numel(), LR, B1, B2,
                                             EPS, _st()), "dr_embed_adam_flush")
        torch.cuda.synchronize()

    def moments(self):
        """(m, v, m_w, v_w, stamps) of the global rows, reassembled from the ranks' state blocks."""
        D, W, total = self.ar.D, self.ar.world, self.ar.total
        m, v = np.zeros((total, D), np.float32), np.zeros((total, D), np.float32)
        mw, vw, stamp = np.zeros(total, np.float32), np.zeros(total, np.float32), np.zeros(total, np.int32)
        for g in range(W):
            n = self.ar.nloc[g]
            st = self.state[g][:n].cpu().numpy()
            m[g::W], v[g::W] = st[:, D:2 * D], st[:, 2 * D:3 * D]
            mw[g::W], vw[g::W] = st[:, 3 * D + 1], st[:, 3 * D + 2]
            stamp[g::W] = st[:, 3 * D + 4].view(np.int32)
            assert (st[:, 3 * D + 3].view(np.int32) == 0).all(), f"rank {g}: a lookup count was left behind"
        return m, v, mw, vw, stamp


def run_world(layout_world, W, rows, D, table, lin, ids_steps, grads, B, hist=HIST):
    """STEPS global steps of W ranks (slices of B examples) on shards laid out for `layout_world` ranks (W, or 1 for
    world 1 running the same slices).  Returns (tables, lin, moments, forward stacks per step)."""
    ar = Arenas(rows, D, layout_world, table, lin)
    rk = Ranks(ar, hist)
    S = len(rows)
    bias = torch.tensor([0.3], device="cuda")
    stacks = []
    sl = lambda t, g: t[g * B:(g + 1) * B]
    for t, (ids_t, (gl_t, gs_t)) in enumerate(zip(ids_steps, grads)):
        rk.clock.advance()
        for g in range(W):
            rk.mark(sl(ids_t, g), B)
        for g in range(layout_world):
            rk.prepare(g)
        stack = torch.empty((W * B, S, D), device="cuda")
        sum_e = torch.empty((W * B, D), device="cuda")
        logit = torch.empty((W * B,), device="cuda")
        for g in range(W):
            fwd(ar, sl(ids_t, g), bias, B, sl(stack, g), sl(sum_e, g), sl(logit, g))
        for g in range(W):
            bwd(rk.grad, sl(ids_t, g), sl(stack, g), sl(sum_e, g), sl(gl_t, g), sl(gs_t, g), None, 1.0 / W, B)
        for g in range(layout_world):
            rk.apply(g)
        torch.cuda.synchronize()
        stacks.append(stack.cpu().numpy())
        gt, gw = rk.grad.gather()           # sentinels intact, and every gradient row cleared by the apply
        assert not gt.any() and not gw.any(), f"step {t + 1}: gradient arena not cleared"
    for g in range(layout_world):
        rk.flush(g)
    tab, lw = ar.gather()
    return tab, lw, rk.moments(), stacks


def dense_adam(table, lin, rows, ids_steps, grads, W, lr=LR):
    """float64 tf.keras Adam applied densely to the unsharded table: every row's m, v decay and every row moves each
    step; the row gradient is the mean over the W slices' lookups (FM part g_logit (sum_e - e) + g_stack).

    Also returns, per row, how far float32 rounding of the gradient can move the row: the sum A of the magnitudes of
    the parts of its contributions (the float32 gradient is off by up to ~1e-5 A in any summation order; a gradient that
    cancels to far below its parts is known only to that absolute accuracy) carried into every later update through m
    and v, lr_t * 1e-5 A / (sqrt(v) + eps) per step and per moment."""
    offs = np.concatenate([[0], np.cumsum(rows)[:-1]])
    P, Lw = table.astype(np.float64), lin.astype(np.float64)
    M, V, Mw, Vw = np.zeros_like(P), np.zeros_like(P), np.zeros_like(Lw), np.zeros_like(Lw)
    gmax = 0.0
    Amax, Amax_w, E, Ew = np.zeros_like(P), np.zeros_like(Lw), np.zeros_like(P), np.zeros_like(Lw)
    omb1, omb2 = np.float64(np.float32(1) - np.float32(B1)), np.float64(np.float32(1) - np.float32(B2))
    for t, (ids, (gl, gs)) in enumerate(zip(ids_steps, grads), start=1):
        ok = (ids >= 0) & (ids < np.array(rows)[None, :])
        r = np.where(ok, ids + offs[None, :], 0)
        e = np.where(ok[..., None], P[r], 0.0)
        d = gl.astype(np.float64)[:, None, None] * (e.sum(1, keepdims=True) - e) + gs.astype(np.float64)
        Gr, Gw = np.zeros_like(P), np.zeros_like(Lw)
        np.add.at(Gr, r[ok], d[ok] / W)
        np.add.at(Gw, r[ok], np.broadcast_to(gl.astype(np.float64)[:, None], ok.shape)[ok] / W)
        A, Aw = np.zeros_like(P), np.zeros_like(Lw)
        # the float32 gradient of one lookup rounds relative to its parts, not to their (possibly cancelling) sum
        parts = (np.abs(gl.astype(np.float64))[:, None, None] * (np.abs(e).sum(1, keepdims=True) + np.abs(e))
                 + np.abs(gs.astype(np.float64)))
        np.add.at(A, r[ok], parts[ok] / W)
        np.add.at(Aw, r[ok], np.abs(np.broadcast_to(gl.astype(np.float64)[:, None], ok.shape)[ok]) / W)
        Amax, Amax_w = np.maximum(Amax, A), np.maximum(Amax_w, Aw)
        gmax = max(gmax, np.abs(Gr).max(), np.abs(Gw).max())
        lt = np.float64(np.float32(lr)) * np.sqrt(1 - np.float64(np.float32(B2)) ** t) / (1 - np.float64(np.float32(B1)) ** t)
        for p, m, v, g in ((P, M, V, Gr), (Lw, Mw, Vw, Gw)):
            m += (g - m) * omb1
            v += (g * g - v) * omb2
            p -= lt * m / (np.sqrt(v) + EPS)
        E += 2 * lt * 1e-5 * Amax / (np.sqrt(V) + EPS)
        Ew += 2 * lt * 1e-5 * Amax_w / (np.sqrt(Vw) + EPS)
    return P, Lw, M, V, Mw, Vw, gmax, E, Ew


def make_steps(rng, rows, W, B, S, D, unique):
    ids_steps, grads = [], []
    for t in range(STEPS):
        if unique:
            from test_gpu_sharded_emulated import unique_ids
            ids = unique_ids(rng, W * B, rows)
            # leave some rows out of some steps: drop a random half of the lookups to OOV ids
            ids[rng.random(ids.shape) < 0.5] = -1
        else:
            ids = zipf_ids(rng, W * B, rows, a=1.2)
        # some steps touch only a few slots, so rows sit out 1, 2 and more than HIST steps
        if t in (1, 2, 3):
            ids[:, (t % len(rows))::2] = -1
        ids_steps.append(ids)
        grads.append((rng.standard_normal(W * B).astype(np.float32),
                      rng.standard_normal((W * B, S, D)).astype(np.float32)))
    return ids_steps, grads


def _dev_steps(ids_steps, grads, id_dtype=np.int64):
    return [_dev(i.astype(id_dtype)) for i in ids_steps], [(_dev(a), _dev(b)) for a, b in grads]


@pytest.mark.parametrize("D", [16, 12, 32])
@pytest.mark.parametrize("world,tname", WORLD_TABLES, ids=WT_IDS)
def test_emulated_sharded_adam_matches_dense_adam(world, tname, D):
    """Zipf ids with duplicates, -1 and out-of-range ids: tables, first-order weights, m and v after flush against
    float64 dense Adam on the unsharded table and global batch."""
    rows, B = TABLES[tname], 37
    S = len(rows)
    rng = np.random.default_rng(world * 31 + D)
    table, lin = make_table(rng, rows, D)
    ids_steps, grads = make_steps(rng, rows, world, B, S, D, unique=False)
    ids_d, grads_d = _dev_steps(ids_steps, grads)
    tab, lw, (m, v, mw, vw, stamp), _ = run_world(world, world, rows, D, table, lin, ids_d, grads_d, B)
    P, Lw, M, V, Mw, Vw, gmax, E, Ew = dense_adam(table, lin, rows, ids_steps, grads, world)
    assert (stamp[np.abs(M).sum(1) > 0] == STEPS).all(), "flush left a row behind the clock"
    # fp32 gradients summed in any order (relative 1e-6 of the contributions), then 6 steps of Adam; a replayed step that
    # fell out of the HIST-long ring takes a rate recomputed in float32 (1 - powf(b2, j) cancels: up to ~1e-4 relative at
    # small j), hence the absolute term of 1e-3 lr -- a missed or doubled step moves a row by about lr
    tol_p = 2e-5 * np.abs(P) + 1e-3 * LR + E
    for name, got, want, tol in (("table", tab, P, tol_p), ("first-order", lw, Lw, 2e-5 * np.abs(Lw) + 1e-3 * LR + Ew),
                                 ("m", m, M, 1e-5 * gmax + 1e-5 * np.abs(M)), ("m_w", mw, Mw, 1e-5 * gmax + 1e-5 * np.abs(Mw)),
                                 ("v", v, V, 1e-5 * gmax ** 2 + 1e-5 * np.abs(V)),
                                 ("v_w", vw, Vw, 1e-5 * gmax ** 2 + 1e-5 * np.abs(Vw))):
        err = np.abs(got.astype(np.float64) - want)
        assert (err <= tol).all(), f"{name}: max err {err.max()} (excess {np.max(err - tol)})"


@pytest.mark.parametrize("id_dtype", [np.int64, np.int32], ids=["i64", "i32"])
@pytest.mark.parametrize("D", [16, 12, 32, 128])
@pytest.mark.parametrize("world,tname", [c for c in WORLD_TABLES if c[0] > 1], ids=[i for i, c in zip(WT_IDS, WORLD_TABLES)
                                                                                  if c[0] > 1])
def test_emulated_sharded_adam_bit_identical_to_world1(world, tname, D, id_dtype):
    """Every row looked up at most once per step: one contribution per gradient row, so the forward's rows after each
    replay, the tables, first-order weights and moments at world W equal world 1 running the same slices bit for bit."""
    rows, B = TABLES[tname], 29
    S = len(rows)
    rng = np.random.default_rng(world * 17 + D)
    table, lin = make_table(rng, rows, D)
    ids_steps, grads = make_steps(rng, rows, world, B, S, D, unique=True)
    ids_d, grads_d = _dev_steps(ids_steps, grads, id_dtype)
    got = run_world(world, world, rows, D, table, lin, ids_d, grads_d, B)
    one = run_world(1, world, rows, D, table, lin, ids_d, grads_d, B)
    for t, (a, b) in enumerate(zip(got[3], one[3])):
        assert np.array_equal(_bits(a), _bits(b)), f"step {t + 1}: forward rows at world {world} != world 1"
    for name, a, b in zip(("table", "first-order"), got[:2], one[:2]):
        assert np.array_equal(_bits(a), _bits(b)), f"{name} at world {world} != world 1"
    for name, a, b in zip(("m", "v", "m_w", "v_w", "stamp"), got[2], one[2]):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), f"{name} != world 1"
    P, Lw, *_, E, Ew = dense_adam(table, lin, rows, ids_steps, grads, world)
    assert (np.abs(got[0] - P) <= 2e-5 * np.abs(P) + 1e-3 * LR + E).all()


def test_shard_adam_entries_reject_bad_arguments_without_launching():
    from deep_recommenders_b200 import _lib as L
    lib = L.load()
    n0 = L.launch_count()
    x = torch.zeros(64, device="cuda")
    i = torch.zeros(64, dtype=torch.int32, device="cuda")
    step = torch.ones(1, dtype=torch.int64, device="cuda")
    rows = torch.tensor([8], dtype=torch.int64, device="cuda")
    offs = torch.zeros(1, dtype=torch.int64, device="cuda")
    peers = torch.tensor([i.data_ptr()], dtype=torch.int64, device="cuda")
    st = _st()
    mark = lambda world=1, ids=i.data_ptr(), idb=4: lib.dr_shard_adam_mark(ids, idb, 8, 1, offs.data_ptr(),
                                                                          rows.data_ptr(), world, peers.data_ptr(),
                                                                          step.data_ptr(), st)
    assert mark(world=0) == -1 and mark(world=65) == -1 and mark(ids=None) == -1 and mark(idb=2) == -1
    prep = lambda D=16, touch=i.data_ptr(), stride=32: lib.dr_shard_adam_prepare(
        touch, 2, i.data_ptr(), i.data_ptr(), D, stride, 0, 1, x.data_ptr(), x.data_ptr(), step.data_ptr(), None, 0,
        LR, B1, B2, EPS, st)
    assert prep(D=130) == -1 and prep(D=6) == -1 and prep(touch=None) == -1 and prep(stride=16) == -1
    app = lambda D=16, grad=x.data_ptr(): lib.dr_shard_adam_apply(i.data_ptr(), i.data_ptr(), 2, D, 32, 0, 1,
                                                                   x.data_ptr(), grad, x.data_ptr(), step.data_ptr(),
                                                                   x.data_ptr(), B1, B2, EPS, st)
    assert app(D=0) == -1 and app(grad=None) == -1
    assert L.launch_count() == n0


# ---- the trainer at world 1 -----------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.fixture(scope="module")
def world1():
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(_free_port())
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    yield
    dist.destroy_process_group()


ROWS1, D1, B1_, UNITS = [300, 7, 50, 1000, 21], 16, 384, [32, 8]


def _sharded(exchange, use_graph=True, seed=3):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.sharded import ShardedDeepFMTrainStep
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(ROWS1)]
    sh = ShardedDeepFMTrainStep(cols, D1, UNITS, batch_size=B1_, lr=LR, seed=seed, device="cuda", exchange=exchange,
                                use_graph=use_graph, optimizer="adam_rows_tf")
    with torch.no_grad():
        sh.emb.lin_view().normal_(0, 0.1, generator=torch.Generator(device="cuda").manual_seed(seed))
    return sh


def _batches(n, seed=0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for _ in range(n):
        # a few slots per step are fully OOV, so rows sit out steps
        ids = torch.stack([torch.randint(-1, r + 1, (B1_,), device="cuda", generator=gen) for r in ROWS1], dim=1)
        out.append((ids, torch.randint(0, 2, (B1_,), device="cuda", generator=gen).float()))
    for k in (1, 2):
        out[k][0][:, k::2] = -1
    return out


def _shard_state(sh):
    """(table [rows, D], first-order [rows], m, v, m_w, v_w) of a world-1 shard (local row = global row)."""
    D = sh.D
    st = sh.state[:sh.emb.local_rows]
    return (sh.emb.weight[:, :D], sh.emb.lin_view(), st[:, D:2 * D], st[:, 2 * D:3 * D], st[:, 3 * D + 1],
            st[:, 3 * D + 2])


def _close(a, b, what, rtol=1e-4, atol=1e-6):
    """Equal up to float32 summation order: Adam carries a rounding difference of a gradient element that cancels to
    near zero into its update at up to lr times its relative size, so the bound is relative to the values' scale."""
    err = (a.double() - b.double()).abs()
    a, b = a.detach(), b.detach()
    tol = rtol * b.double().abs() + atol * max(1.0, float(b.double().abs().max()))
    assert bool((err <= tol).all()), f"{what}: max err {float(err.max())}"


@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_world1_sharded_adam_equals_single_gpu_adam_rows_tf(world1, exchange):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    D = D1
    sh = _sharded(exchange).capture()
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(ROWS1)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=UNITS, seed=3, device="cuda", sparse_lr=LR)
    ref = DeepFMTrainStep(model, batch_size=B1_, lr=LR, use_graph=False, optimizer="adam_rows_tf")
    with torch.no_grad():
        model.embeddings.emb_view().copy_(sh.emb.weight[:, :D])
        model.embeddings.lin_view().copy_(sh.emb.lin_view())
        model.embeddings.bias.copy_(sh.bias)
        for i in range(len(ref.layers)):
            ref.w[i].copy_(sh.w[i])
            ref.b[i].copy_(sh.b[i])
    for it, (ids, lab) in enumerate(_batches(6)):
        l_sh = float(sh.step(ids, lab).item())
        l_ref = float(ref.step(ids, lab).item())
        sh.check_overflow()
        assert abs(l_sh - l_ref) <= 1e-5 * abs(l_ref), (it, l_sh, l_ref)
        if it == 0:
            assert torch.equal(sh.stack, ref.stack)
    sh.flush_optimizer()
    ref.flush_optimizer()
    torch.cuda.synchronize()
    c = model.embeddings
    rst = ref.state
    want = (c.emb_view(), c.lin_view(), rst[:, D:2 * D], rst[:, 2 * D:3 * D], rst[:, 3 * D + 1], rst[:, 3 * D + 2])
    for name, a, b in zip(("table", "first-order", "m", "v", "m_w", "v_w"), _shard_state(sh), want):
        _close(a, b, name)
    for i in range(len(ref.layers)):
        _close(sh.w[i], ref.w[i], f"w{i}")
        _close(sh.b[i], ref.b[i], f"b{i}")
    _close(sh.bias, c.bias, "bias")
    n = ref.m_flat.numel()
    _close(sh.m_flat[4:4 + n], ref.m_flat, "tower m")
    _close(sh.v_flat[4:4 + n], ref.v_flat, "tower v")
    _close(sh.m_flat[:1], ref.m_bias, "bias m")
    _close(sh.v_flat[:1], ref.v_bias, "bias v")


@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_world1_sharded_adam_graph_equals_eager_and_capture_is_side_effect_free(world1, exchange):
    g, e = _sharded(exchange, use_graph=True), _sharded(exchange, use_graph=False)
    before = [t.clone() for t in g._persistent_state()]
    g.capture()
    for t, b in zip(g._persistent_state(), before):
        assert torch.equal(t, b), "capture() changed the trainer's state"
    e.capture()
    for ids, lab in _batches(4, seed=1):
        lg, le = float(g.step(ids, lab).item()), float(e.step(ids, lab).item())
        assert abs(lg - le) <= 1e-6 * abs(le), (lg, le)
    g.flush_optimizer()
    e.flush_optimizer()
    for name, a, b in zip(("table", "first-order", "m", "v", "m_w", "v_w"), _shard_state(g), _shard_state(e)):
        _close(a, b, name)
    _close(g.flat, e.flat, "tower")


@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_world1_sharded_adam_save_load_continue(world1, exchange, tmp_path):
    a = _sharded(exchange).capture()
    batches = _batches(5, seed=2)
    for ids, lab in batches[:3]:
        a.step(ids, lab)
    prefix = str(tmp_path / "ck")
    a.save(prefix)
    b = _sharded(exchange, seed=9).capture()
    b.step(*batches[4])                       # b has trained on something else: load must replace all of it
    b.load(prefix)
    assert int(b.clock.step) == int(a.clock.step) == 3
    for ids, lab in batches[3:]:
        la, lb = float(a.step(ids, lab).item()), float(b.step(ids, lab).item())
        assert abs(la - lb) <= 1e-6 * abs(la), (la, lb)
    a.flush_optimizer()
    b.flush_optimizer()
    for name, x, y in zip(("table", "first-order", "m", "v", "m_w", "v_w"), _shard_state(a), _shard_state(b)):
        _close(x, y, name)
    _close(a.flat, b.flat, "tower")
    _close(a.m_flat, b.m_flat, "tower m")
    # an SGD trainer refuses the Adam checkpoint
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.sharded import ShardedDeepFMTrainStep
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(ROWS1)]
    sgd = ShardedDeepFMTrainStep(cols, D1, UNITS, batch_size=B1_, lr=LR, seed=3, device="cuda", exchange=exchange)
    with pytest.raises(ValueError, match="optimizer"):
        sgd.load(prefix)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_world2_sharded_adam_matches_unsharded():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "sharded_adam_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "SHARDED_ADAM_OK" in r.stdout
