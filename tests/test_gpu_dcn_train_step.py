"""DCNTrainStep (the whole-step CUDA-graph trainer of the DCN model) and the two C-ABI entries it adds:
dr_cross_bwd_acc (Cross backward that accumulates the x0 gradient in place) and dr_dcn_head_bce_fwd_bwd (the DCN tail,
Dense(1) on [x_cross | deep] + sigmoid cross-entropy + backward, without the concat).

Single kernels are held to |a - b| <= 1e-5 * sum|terms| + tiny, whole-step compositions to the 1e-4 * scale bound of
test_gpu_assembled_models.test_dcn_step_matches_oracle (float64 compositions of the oracle's layer restatements).
"""
import numpy as np
import pytest
import torch

from oracle import reference_np as R

pytestmark = pytest.mark.gpu

F64 = np.float64


def npy(t):
    return t.detach().cpu().numpy()


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def P(t):
    return None if t is None else t.data_ptr()


@pytest.fixture(params=["ffma", "tc", "tc2", "tc2pair"])
def gemm_variant(request):
    """The GEMM cores the Dense / Cross tests of test_gpu_dense_cross.py run under."""
    from deep_recommenders_b200 import _lib
    pair_default = _lib.tune_get("tc_pair")
    if request.param == "tc":
        _lib.enable_tensor_core_gemm(variant=1)
    elif request.param.startswith("tc2"):
        _lib.enable_tensor_core_gemm(variant=2)
        if request.param != "tc2":
            _lib.tune("tc_pair", 2)
    else:
        _lib.disable_tensor_core_gemm()
    yield request.param
    _lib.tune("tc_pair", pair_default)
    _lib.enable_tensor_core_gemm()


# ---- 1. dr_cross_bwd_acc ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 513])
@pytest.mark.parametrize("d", [12, 30, 832])            # 30: rows not a multiple of 4 wide -> the scalar prologue
@pytest.mark.parametrize("x_is_x0", [0, 1])
@pytest.mark.parametrize("use_bias", [True, False])
@pytest.mark.parametrize("alpha", [0.0, 0.1])
@pytest.mark.parametrize("low_rank", [False, True])
def test_cross_bwd_acc_matches_cross_bwd_plus_adds(gemm_variant, lib, low_rank, alpha, use_bias, x_is_x0, d, B):
    from deep_recommenders_b200 import _lib
    from deep_recommenders_b200._lib import check
    r = {12: 4, 30: 6, 832: 64}[d] if low_rank else 0
    _lib.ensure_gemm_workspace(B, d, d, "cuda")
    rng = np.random.default_rng(B + d + r)
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    x0 = cu(f(B, d))
    x = x0 if x_is_x0 else cu(f(B, d))
    w = None if r else cu(f(d, d) / np.float32(np.sqrt(d)))
    uk = cu(f(d, r) / np.float32(np.sqrt(d))) if r else None
    vk = cu(f(r, d) / np.float32(np.sqrt(r))) if r else None
    b = cu(0.1 * f(d)) if use_bias else None
    g = cu(f(B, d))
    pre = cu(f(B, d))
    st = torch.cuda.current_stream().cuda_stream
    e = lambda *s: torch.empty(s, device="cuda", dtype=torch.float32)
    u, y, xu = e(B, d), e(B, d), (e(B, r) if r else None)
    check(lib.dr_cross_fwd(P(x0), P(x), P(w), P(uk), P(vk), P(b), alpha, B, d, r, P(xu), P(u), P(y), st), "dr_cross_fwd")

    def grads():
        return dict(h=e(B, d), t=e(B, r) if r else None, gx=e(B, d), gw=None if r else e(d, d), guk=e(d, r) if r else None,
                    gvk=e(r, d) if r else None, gb=e(d) if use_bias else None)

    a, c = grads(), grads()
    gx0_ref = e(B, d)
    check(lib.dr_cross_bwd(P(x0), P(x), P(w), P(uk), P(vk), alpha, P(u), P(xu), P(g), B, d, r, P(a["h"]), P(a["t"]),
                           P(gx0_ref), P(a["gx"]), P(a["gw"]), P(a["guk"]), P(a["gvk"]), P(a["gb"]), st), "dr_cross_bwd")
    gx0 = pre.clone()
    c["gx"].fill_(float("nan"))
    check(lib.dr_cross_bwd_acc(P(x0), P(x), P(w), P(uk), P(vk), alpha, P(u), P(xu), P(g), B, d, r, P(c["h"]), P(c["t"]),
                               P(gx0), None if x_is_x0 else P(c["gx"]), P(c["gw"]), P(c["guk"]), P(c["gvk"]), P(c["gb"]),
                               x_is_x0, st), "dr_cross_bwd_acc")
    torch.cuda.synchronize()
    assert torch.equal(a["h"], c["h"]), "h differs from the existing prologue's"
    terms = [npy(pre).astype(F64), npy(gx0_ref).astype(F64)]
    if x_is_x0:
        terms.append(npy(a["gx"]).astype(F64))
        assert torch.isnan(c["gx"]).all(), "gx written although x_is_x0 was set"
    else:
        assert torch.equal(a["gx"], c["gx"])
    want, scale = sum(terms), sum(np.abs(t) for t in terms)
    err = np.abs(npy(gx0).astype(F64) - want)
    assert (err <= 1e-5 * scale + 1e-7).all(), err.max()
    # parameter gradients: same GEMMs as dr_cross_bwd (split-K reductions: equal up to summation order)
    ah, ax = np.abs(npy(a["h"])).astype(F64), np.abs(npy(x)).astype(F64)
    scales = {"gb": ah.sum(0)}
    if r:
        scales["gvk"] = np.abs(npy(xu)).astype(F64).T @ ah
        scales["guk"] = ax.T @ (ah @ np.abs(npy(vk)).astype(F64).T)
    else:
        scales["gw"] = ax.T @ ah
    for k, sc in scales.items():
        if a[k] is None:
            continue
        err = np.abs(npy(a[k]).astype(F64) - npy(c[k]).astype(F64))
        assert (err <= 1e-5 * sc + 1e-7).all(), (k, err.max())


def test_cross_bwd_acc_validates_before_launch(lib):
    z = None
    # x_is_x0 without gx0 / with x != x0; gx missing on an upper layer; full rank without W
    assert lib.dr_cross_bwd_acc(16, 16, 16, z, z, 0.0, 16, z, 16, 4, 8, 0, 16, z, z, z, 16, z, z, z, 1, z) == -1
    assert lib.dr_cross_bwd_acc(16, 32, 16, z, z, 0.0, 16, z, 16, 4, 8, 0, 16, z, 16, z, 16, z, z, z, 1, z) == -1
    assert lib.dr_cross_bwd_acc(16, 32, 16, z, z, 0.0, 16, z, 16, 4, 8, 0, 16, z, 16, z, 16, z, z, z, 0, z) == -1
    assert lib.dr_cross_bwd_acc(16, 16, z, z, z, 0.0, 16, z, 16, 4, 8, 0, 16, z, 16, z, 16, z, z, z, 1, z) == -1
    assert b"full-rank" in lib.dr_last_error()


# ---- 2. dr_dcn_head_bce_fwd_bwd -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 513])
@pytest.mark.parametrize("act", [None, "relu"])
@pytest.mark.parametrize("d,n", [(8, 4), (832, 128), (3968, 128), (30, 7)])      # (30, 7): the scalar form
@pytest.mark.parametrize("nullable", [False, True])
def test_dcn_head_matches_float64(lib, nullable, d, n, act, B):
    from deep_recommenders_b200 import ops
    from deep_recommenders_b200._lib import check
    rng = np.random.default_rng(B + d + n)
    xc = rng.standard_normal((B, d)).astype(np.float32)
    deep = rng.standard_normal((B, n)).astype(np.float32)
    if act == "relu":
        deep = np.maximum(deep, 0)
    w = (rng.standard_normal(d + n) / np.sqrt(d + n)).astype(np.float32)
    bias = np.float32(0.3)
    y = rng.integers(0, 2, B).astype(np.float32)
    e = lambda *s: torch.full(s, float("nan"), device="cuda", dtype=torch.float32)
    out = dict(logit=e(B), prob=e(B), loss=e(1), g_logit=e(B), g_xc=e(B, d), g_deep=e(B, n), gw=e(d + n), gb=e(1), gb_deep=e(n))
    if nullable:
        for k in ("logit", "prob", "g_logit", "g_xc", "gw", "gb", "gb_deep"):
            out[k] = None
    xct, dt, wt, bt, yt = cu(xc), cu(deep), cu(w), cu(np.array([bias])), cu(y)
    check(lib.dr_dcn_head_bce_fwd_bwd(P(xct), P(dt), P(wt), P(bt), P(yt), B, d, n, ops.act_code(act), P(out["logit"]),
                                      P(out["prob"]), P(out["loss"]), P(out["g_logit"]), P(out["g_xc"]), P(out["g_deep"]),
                                      P(out["gw"]), P(out["gb"]), P(out["gb_deep"]), torch.cuda.current_stream().cuda_stream),
          "dr_dcn_head_bce_fwd_bwd")
    torch.cuda.synchronize()
    feat = np.concatenate([xc, deep], 1).astype(F64)
    w64 = w.astype(F64)
    z = feat @ w64 + F64(bias)
    zs = np.abs(feat) @ np.abs(w64) + abs(F64(bias))
    p = 1 / (1 + np.exp(-z))
    gl = (p - y) / B
    gl_tol = 1e-5 * (1 + zs) / B                      # d sigmoid / dz <= 1/4: the logit's rounding carried into g
    loss = np.mean(np.maximum(z, 0) - z * y + np.log1p(np.exp(-np.abs(z))))
    mask = (deep > 0).astype(F64) if act == "relu" else np.ones_like(deep, dtype=F64)
    want = dict(logit=(z, 1e-5 * zs), prob=(p, 1e-5 * (1 + zs)), loss=(loss, 1e-5 * (abs(loss) + zs.mean())),
                g_logit=(gl, gl_tol),
                g_xc=(gl[:, None] * w64[None, :d], gl_tol[:, None] * np.abs(w64[None, :d])),
                g_deep=(gl[:, None] * w64[None, d:] * mask, gl_tol[:, None] * np.abs(w64[None, d:])),
                gw=(feat.T @ gl, np.abs(feat).T @ (1e-5 * np.abs(gl) + gl_tol)),
                gb=(gl.sum(), 1e-5 * np.abs(gl).sum() + gl_tol.sum()),
                gb_deep=((gl[:, None] * w64[None, d:] * mask).sum(0), (1e-5 * np.abs(gl) + gl_tol) @ np.ones((B, 1)) * np.abs(w64[d:])))
    for k, (ref, tol) in want.items():
        if out[k] is None:
            continue
        got = npy(out[k]).astype(F64).reshape(np.shape(ref))
        assert (np.abs(got - ref) <= tol + 1e-7).all(), (k, np.abs(got - ref).max())


def test_dcn_head_wider_than_served_is_enotsup(lib):
    rc = lib.dr_dcn_head_bce_fwd_bwd(16, 16, 16, None, 16, 4, 4000, 128, 1, None, None, 16, None, None, None, None, None,
                                     None, None)
    assert rc == -3 and b"4128" in lib.dr_last_error()
    assert lib.dr_dcn_head_bce_fwd_bwd(16, 16, 16, None, 16, 4, 8, 4, 9, None, None, 16, None, None, None, None, None, None,
                                       None) == -1


# ---- float64 oracle of one DCN training step ----------------------------------------------------------------------------
def _dnn_backward(hs, ws, g_out, acts):
    """float64 backward through Dense layers given hs = [input, h1, ..., h_last] and the upstream gradient of h_last.
    Returns (g_input, gws, gbs, scales of gws, scales of gbs); the scales are the sums of |terms| of every dot product."""
    gws, gbs, sws, sbs = [], [], [], []
    g = g_out
    for i in range(len(ws) - 1, -1, -1):
        gx, gw, gb = R.dense_grad(hs[i], ws[i], hs[i + 1], g, acts[i], F64)
        gz = np.abs(g * (hs[i + 1] > 0)) if acts[i] == "relu" else np.abs(g)
        gws.append(gw)
        gbs.append(gb)
        sws.append(np.abs(hs[i]).T @ gz)
        sbs.append(gz.sum(0))
        g = gx
    return g, gws[::-1], gbs[::-1], sws[::-1], sbs[::-1]


def _param_names(model):
    names = {}
    for i, c in enumerate(model.cross):
        for k in ("kernel", "kernel_u", "kernel_v", "bias"):
            if getattr(c, k) is not None:
                names[f"cross.{i}.{k}"] = getattr(c, k)
    for i, l in enumerate(model.dnn.layers):
        names[f"dnn.{i}.kernel"], names[f"dnn.{i}.bias"] = l.kernel, l.bias
    names["head.kernel"], names["head.bias"] = model.head.kernel, model.head.bias
    return names


def _oracle_step(model, ids, y, alpha):
    """loss (mean), prob, sum|terms| of every logit, {parameter: (gradient, scale)}, per-table gradient of the mean BCE,
    the tables before the step; all float64."""
    coll = model.embeddings
    S, D = coll.num_slots, coll.dim
    B = ids.shape[0]
    tables = [npy(coll.table(s)) for s in range(S)]
    x0 = R.stack_embeddings(tables, ids).reshape(B, S * D).astype(F64)
    g64 = lambda t: None if t is None else npy(t).astype(F64)
    cp = [(g64(c.kernel), g64(c.kernel_u), g64(c.kernel_v), g64(c.bias)) for c in model.cross]
    xs = [x0]
    for w, u, v, b in cp:
        xs.append(R.cross(x0, xs[-1], w, b, u, v, alpha, F64)[0])
    dw = [g64(l.kernel) for l in model.dnn.layers]
    db = [g64(l.bias) for l in model.dnn.layers]
    acts = [l.activation for l in model.dnn.layers]
    hs = [x0]
    for w, b, a in zip(dw, db, acts):
        hs.append(R.dense(hs[-1], w, b, a, F64))
    hw, hb = g64(model.head.kernel), g64(model.head.bias)
    feat = np.concatenate([xs[-1], hs[-1]], 1)
    z = feat @ hw + hb
    p = 1 / (1 + np.exp(-z))
    loss = float(np.mean(np.maximum(z, 0) - z * y + np.log1p(np.exp(-np.abs(z)))))
    gz = (p - y) / B
    g_feat = gz @ hw.T
    d = S * D
    zs = (np.abs(feat) @ np.abs(hw) + np.abs(hb)).reshape(-1)
    grads = {"head.kernel": (feat.T @ gz, np.abs(feat).T @ np.abs(gz)), "head.bias": (gz.sum(0), np.abs(gz).sum(0))}
    g_x0, gws, gbs, sws, sbs = _dnn_backward(hs, dw, g_feat[:, d:], acts)
    for i in range(len(dw)):
        grads[f"dnn.{i}.kernel"], grads[f"dnn.{i}.bias"] = (gws[i], sws[i]), (gbs[i], sbs[i])
    g = g_feat[:, :d]
    for i in range(len(cp) - 1, -1, -1):
        w, u, v, b = cp[i]
        gr = R.cross_grad(x0, xs[i], g, w, u, v, b, alpha, F64)
        for k, name in (("gw", "kernel"), ("gu", "kernel_u"), ("gv", "kernel_v"), ("gb", "bias")):
            if k in gr and getattr(model.cross[i], name) is not None:
                grads[f"cross.{i}.{name}"] = (gr[k], np.abs(gr[k]).max())
        g_x0 = g_x0 + gr["gx0"]
        g = gr["gx"]
    g_x0 = g_x0 + g                                           # xs[0] is x0 itself
    g_tab = [np.zeros_like(t, dtype=F64) for t in tables]
    g3 = g_x0.reshape(B, S, D)
    for s in range(S):
        ok = ids[:, s] >= 0
        np.add.at(g_tab[s], ids[ok, s], g3[ok, s])
    return loss, p.reshape(-1), zs, grads, g_tab, tables


def _make_model(rows, D, units, ncross, alpha, proj=None, seed=5, B=8):
    """A built DCN with non-zero biases (zero-init biases would hide bias-path errors)."""
    from deep_recommenders.keras.layers import DCN
    model = DCN(rows, D, num_cross=ncross, dnn_units=units, diag_scale=alpha, projection_dim=proj, seed=seed, device="cuda")
    model.logits(torch.zeros((B, len(rows)), dtype=torch.int64, device="cuda"))
    gen = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for layer in list(model.cross) + list(model.dnn.layers) + [model.head]:
            layer.bias.copy_(0.1 * torch.randn(layer.bias.shape, device="cuda", generator=gen))
    return model


def _batch(rng, rows, B, oov=True):
    ids = np.stack([rng.integers(-1 if oov else 0, r, B) for r in rows], axis=1).astype(np.int64)
    return ids, rng.integers(0, 2, (B, 1)).astype(np.float32)


# ---- 3. one trainer step against the oracle -----------------------------------------------------------------------------
@pytest.mark.parametrize("B,S,D,units,ncross,alpha,proj,id_dtype,hot", [
    (200, 6, 8, [32, 16], 2, 0.0, None, torch.int64, False),
    (513, 26, 32, [64, 32, 16], 3, 0.1, None, torch.int64, False),     # C3-shaped: d = 832, 3 Cross layers
    (300, 6, 8, [32, 16], 2, 0.1, 8, torch.int64, False),              # low rank
    (1200, 4, 8, [16], 1, 0.0, None, torch.int64, True),               # OOV ids and one id repeated 1000 times
    (200, 6, 8, [32, 16], 2, 0.0, None, torch.int32, False),
])
def test_one_step_matches_oracle(B, S, D, units, ncross, alpha, proj, id_dtype, hot):
    from deep_recommenders_b200 import DCNTrainStep
    rows = [97 + 3 * i for i in range(S)]
    model = _make_model(rows, D, units, ncross, alpha, proj)
    ids, y = _batch(np.random.default_rng(B + S), rows, B)
    if hot:
        ids[:1000, 0] = 7
        ids[1000:1010, 1] = -1
    loss_ref, p_ref, zs, grads, g_tab, tables = _oracle_step(model, ids, y, alpha)
    lr = 1.0       # one step only: p - g keeps every bit of g that fp32 can hold next to p
    tr = DCNTrainStep(model, batch_size=B, lr=lr, id_dtype=id_dtype).capture()
    before = {k: npy(p).astype(F64) for k, p in _param_names(model).items()}
    loss = tr.step(torch.from_numpy(ids).cuda().to(id_dtype), cu(y))
    torch.cuda.synchronize()
    assert abs(float(loss) - loss_ref) <= 1e-5 * abs(loss_ref) + 1e-6
    assert (np.abs(npy(tr.prob) - p_ref) <= 2e-5 * (1 + zs)).all()
    ulp = 2.0 ** -23
    for k, p in _param_names(model).items():
        ref, sc = grads[k]
        after = npy(p).astype(F64)
        got = (before[k] - after) / lr
        tol = 1e-4 * sc + 1e-6 + ulp * (np.abs(before[k]) + np.abs(after)) / lr
        assert (np.abs(got - ref.reshape(got.shape)) <= tol).all(), (k, np.abs(got - ref.reshape(got.shape)).max())
    for s in range(S):
        after = npy(model.embeddings.table(s)).astype(F64)
        got = (tables[s].astype(F64) - after) / lr
        tol = 1e-4 * np.abs(g_tab[s]).max() + 1e-6 + ulp * (np.abs(tables[s]) + np.abs(after)) / lr
        assert (np.abs(got - g_tab[s]) <= tol).all(), ("table", s)


# ---- 4. three steps against the autograd path ---------------------------------------------------------------------------
def _autograd_steps(model, batches, lr):
    from deep_recommenders_b200 import ops
    model.embeddings.sparse_lr = lr                          # fused row-sparse SGD in the embedding backward
    dense = [p for n, p in model.named_parameters() if not n.startswith("embeddings.")]
    losses = []
    for ids, y in batches:
        z = model.logits(ids)
        loss, gz, _ = ops.bce_with_logits(z, y)
        z.backward(gz.view_as(z))
        with torch.no_grad():
            for p in dense:
                ops.sgd_step_(p, p.grad, lr)
                p.grad = None
        losses.append(float(loss))
    return losses


def _three_batches(rows, B, seed=11):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(3):
        ids, y = _batch(rng, rows, B)
        out.append((torch.from_numpy(ids).cuda(), cu(y)))
    return out


def _assert_params_agree(m_a, m_b, init, rtol):
    pa, pb = _param_names(m_a), _param_names(m_b)
    pa["tables"], pb["tables"] = m_a.embeddings.weight, m_b.embeddings.weight
    for k in pa:
        a, b = npy(pa[k]).astype(F64), npy(pb[k]).astype(F64)
        moved = np.abs(b - init[k]).max()
        assert moved > 0, f"{k} did not train"
        assert np.abs(a - b).max() <= rtol * moved + 1e-7, (k, np.abs(a - b).max(), moved)


def _snapshot(model):
    s = {k: npy(p).astype(F64).copy() for k, p in _param_names(model).items()}
    s["tables"] = npy(model.embeddings.weight).astype(F64).copy()
    return s


@pytest.mark.parametrize("proj", [None, 8])
def test_three_steps_match_the_autograd_path(proj):
    from deep_recommenders_b200 import DCNTrainStep
    B, S, D, lr = 257, 6, 8, 0.05
    rows = [97 + 3 * i for i in range(S)]
    m_tr = _make_model(rows, D, [32, 16], 2, 0.1, proj)
    m_ag = _make_model(rows, D, [32, 16], 2, 0.1, proj)      # same seed: the same initial weights
    init = _snapshot(m_ag)
    batches = _three_batches(rows, B)
    want = _autograd_steps(m_ag, batches, lr)
    tr = DCNTrainStep(m_tr, batch_size=B, lr=lr).capture()
    got = [float(tr.step(i, y)) for i, y in batches]
    for a, b in zip(got, want):
        assert abs(a - b) <= 1e-5 * abs(b) + 1e-6
    _assert_params_agree(m_tr, m_ag, init, 1e-4)


# ---- 5. graph replay == eager launches; capture() is side-effect free ----------------------------------------------------
def test_graph_equals_eager_and_capture_leaves_parameters_alone():
    from deep_recommenders_b200 import DCNTrainStep
    B, S, D, lr = 257, 6, 8, 0.05
    rows = [97 + 3 * i for i in range(S)]
    m_g, m_e = (_make_model(rows, D, [32, 16], 2, 0.1) for _ in range(2))
    init = _snapshot(m_e)
    t_g = DCNTrainStep(m_g, batch_size=B, lr=lr, use_graph=True)
    t_e = DCNTrainStep(m_e, batch_size=B, lr=lr, use_graph=False)
    ids0, y0 = _three_batches(rows, B, seed=3)[0]
    for t in (t_g, t_e):
        t.ids.copy_(ids0)                                   # capture()'s warm-up step runs on real ids
        t.labels.copy_(y0.reshape(-1))
        state = [x.clone() for x in t._persistent_state()]
        assert t.launches_per_step is None
        t.capture()
        for x, keep in zip(t._persistent_state(), state):
            assert torch.equal(x, keep), "capture() changed a parameter"
    assert t_g.graph is not None and t_e.graph is None
    assert t_g.launches_per_step == t_e.launches_per_step and t_g.launches_per_step > 0
    batches = _three_batches(rows, B)
    for i, y in batches:
        lg, le = float(t_g.step(i, y)), float(t_e.step(i, y))
        assert abs(lg - le) <= 1e-5 * abs(le) + 1e-6
    n = t_e.launches_per_step
    from deep_recommenders_b200 import _lib
    c0 = _lib.launch_count()
    t_e.step(*batches[0])
    assert _lib.launch_count() - c0 == n, "launches per step changed between steps"
    t_g.step(*batches[0])
    _assert_params_agree(m_g, m_e, init, 1e-4)


# ---- 6. fit_host == blocking train_step_host calls ----------------------------------------------------------------------
def test_fit_host_returns_every_loss():
    from deep_recommenders_b200 import DCNTrainStep
    B, S, D, lr = 128, 6, 8, 0.05
    rows = [97 + 3 * i for i in range(S)]
    rng = np.random.default_rng(2)
    host = []
    for _ in range(5):
        ids, y = _batch(rng, rows, B)
        host.append((torch.from_numpy(ids).pin_memory(), torch.from_numpy(y).pin_memory()))
    t_a = DCNTrainStep(_make_model(rows, D, [32, 16], 2, 0.1), batch_size=B, lr=lr).capture()
    t_b = DCNTrainStep(_make_model(rows, D, [32, 16], 2, 0.1), batch_size=B, lr=lr).capture()
    got = t_a.fit_host(host)
    want = [t_b.train_step_host(*bt) for bt in host]
    assert len(got) == 5
    for a, b in zip(got, want):
        assert abs(a - b) <= 1e-5 * abs(b) + 1e-6
    assert len(set(want)) == 5                               # distinct batches: a repeated loss would be a stale read


# ---- 7. the model's parameters alias the trainer's flat buffer ----------------------------------------------------------
def test_layer_api_sees_the_trained_weights():
    from deep_recommenders_b200 import DCNTrainStep
    B, S, D = 200, 6, 8
    rows = [97 + 3 * i for i in range(S)]
    model = _make_model(rows, D, [32, 16], 2, 0.1)
    init = _snapshot(model)
    (ids, y), (ids2, y2), _ = _three_batches(rows, B)
    tr = DCNTrainStep(model, batch_size=B, lr=0.5).capture()
    tr.step(ids, y)
    torch.cuda.synchronize()
    for k, p in _param_names(model).items():
        assert p.data_ptr() >= tr.flat.data_ptr() and p.data_ptr() < tr.flat.data_ptr() + tr.flat.numel() * 4, k
        assert np.abs(npy(p).astype(F64) - init[k]).max() > 0, f"{k} did not train"
    with torch.no_grad():
        z = npy(model.logits(ids2)).reshape(-1).astype(F64)  # layer API, on the weights the step left behind
    tr.step(ids2, y2)                                         # the trainer's forward reads those same weights
    got = npy(tr.logit).astype(F64)
    assert np.abs(got - z).max() <= 2e-5 * (1 + np.abs(z).max())


# ---- 8. constructor errors ----------------------------------------------------------------------------------------------
def test_constructor_errors():
    from deep_recommenders.keras.layers import DCN
    from deep_recommenders_b200 import DCNTrainStep
    from deep_recommenders_b200._lib import DeepRecError
    with pytest.raises(DeepRecError, match="CUDA"):
        DCNTrainStep(DCN([10, 10], 8, num_cross=1, dnn_units=[8], device="cpu"), batch_size=4)
    with pytest.raises(ValueError, match="DNN"):
        DCNTrainStep(DCN([10, 10], 8, num_cross=1, dnn_units=[], device="cuda"), batch_size=4)
    with pytest.raises(ValueError, match="Cross layer"):
        DCNTrainStep(DCN([10, 10], 8, num_cross=0, dnn_units=[8], device="cuda"), batch_size=4)
    reg = DCN([10, 10], 8, num_cross=2, dnn_units=[8], device="cuda")
    reg.cross[1]._kernel_regu = lambda w: (w * w).sum()
    with pytest.raises(ValueError, match="regulariser"):
        DCNTrainStep(reg, batch_size=4)
    with pytest.raises(ValueError, match="head"):
        DCNTrainStep(DCN([5] * 33, 128, num_cross=1, dnn_units=[8], device="cuda"), batch_size=4)   # d = 4224
