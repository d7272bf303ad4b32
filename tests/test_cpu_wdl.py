"""CPU checks of Wide & Deep (run with -m "not gpu"): the host twin of the crossing against the independent Python
restatement, crossed_column / FtrlOptimizer validation, the oracle against the reference's own model, the row-sparse
FTRL against TensorFlow's dense update, and the C-ABI rejections of the wide entries."""
import ctypes as C
import os

import numpy as np
import pytest

import wdl_oracle as W

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wdl_golden.npz")
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def _host_cross(keys, B, N, hash_key=W.DEFAULT_HASH_KEY):
    """keys: per key, a per-example list of raw values (ints or strings); ragged when any list is not length 1."""
    from deep_recommenders_b200.hashing import _cross_key_host, cross_hash_host
    from deep_recommenders_b200.feature_column import RaggedFeature
    packed = []
    for per_ex in keys:
        flat = [v for vals in per_ex for v in vals]
        arr = np.asarray(flat, dtype=np.int64) if all(isinstance(v, int) for v in flat) and flat else flat
        if all(len(v) == 1 for v in per_ex):
            packed.append(_cross_key_host(arr if isinstance(arr, np.ndarray) else np.asarray(flat, dtype=object)))
        else:
            splits = np.cumsum([0] + [len(v) for v in per_ex])
            vals = arr if isinstance(arr, np.ndarray) else (np.asarray(flat, dtype=object) if flat else
                                                            np.zeros(0, dtype=np.int64))
            packed.append(_cross_key_host(RaggedFeature(vals, splits)))
    return cross_hash_host(packed, B, N, hash_key)


def test_fingerprint_cat64_restatements_agree():
    from deep_recommenders_b200 import build
    build.build()
    # two single-valued int keys: the host twin's [B] path equals the chained Python FingerprintCat64
    a, b = [[0], [1], [-2], [I64_MAX], [I64_MIN], [12345]], [[7], [0], [3], [I64_MIN], [-5], [1 << 40]]
    ids, splits = _host_cross([a, b], 6, (1 << 62) + 11)
    assert splits is None
    want = [W.cross_example([x, y], (1 << 62) + 11)[0] for x, y in zip(a, b)]
    assert ids.tolist() == want


@pytest.mark.parametrize("case", ["strings", "mixed", "empty", "minus_one", "multi", "three", "order", "hash_key"])
def test_host_crossing_matches_python(case):
    rng = np.random.default_rng(3)
    B, N = 9, 1000003
    s = [["F"], ["M"], [""], ["ab" * 20], ["x"], ["hello"], ["M"], ["F"], ["é"]]
    i = [[1], [18], [25], [-1], [-7], [I64_MAX], [I64_MIN], [0], [56]]
    hk = W.DEFAULT_HASH_KEY
    if case == "strings":
        keys = [s, [["a"], ["b"], ["c"], ["d"], ["e"], ["f"], ["g"], ["h"], ["i"]]]
    elif case == "mixed":
        keys = [s, i]
    elif case == "empty":
        keys = [[[]] * B, i]
    elif case == "minus_one":
        keys = [i, [[-1]] * 3 + [[4]] * 6]
    elif case == "multi":
        keys = [[[int(x) for x in rng.integers(-2, 5, int(rng.integers(0, 4)))] for _ in range(B)],
                [["u", "", "v"], [], ["w"], ["x", "y"], ["z"], [""], ["a", "a"], ["b"], ["c", "d", "e"]]]
    elif case == "three":
        keys = [s, i, [["p", "q"]] * B]
    elif case == "order":
        keys = [i, s]
    else:
        keys, hk = [s, i], 0x1234567
    got, splits = _host_cross(keys, B, N, hk)
    want_ids, want_splits = W.cross_batch(keys, N, hk)
    if splits is None:
        per_ex = [want_ids[want_splits[b]:want_splits[b + 1]].tolist() for b in range(B)]
        assert got.tolist() == [p[0] if p else -1 for p in per_ex]
        assert all(len(p) <= 1 for p in per_ex)
    else:
        assert splits.tolist() == want_splits.tolist()
        assert got.tolist() == want_ids.tolist()


def test_key_order_changes_the_cross():
    a, b = [["F"], ["M"]], [[18], [25]]
    ab, _ = _host_cross([a, b], 2, 1 << 40)
    ba, _ = _host_cross([b, a], 2, 1 << 40)
    assert (ab != ba).all()


def test_crossed_column_validation():
    from deep_recommenders_b200 import feature_column as fc
    with pytest.raises(ValueError):
        fc.crossed_column(["a"], 10)
    with pytest.raises(ValueError):
        fc.crossed_column(["a", "b"], 0)
    with pytest.raises(NotImplementedError):
        fc.crossed_column([fc.categorical_column_with_identity("a", 3), "b"], 10)
    with pytest.raises(NotImplementedError):
        fc.crossed_column([fc.crossed_column(["a", "b"], 10), "c"], 10)
    c = fc.crossed_column(["user_gender", "user_age"], 14)
    assert c.name == "user_age_X_user_gender" and c.num_buckets == 14 and c.hash_key == 0xDECAFCAFFE
    assert fc.indicator_column(c).name == "user_age_X_user_gender_indicator"


def test_ftrl_optimizer_validation():
    from deep_recommenders_b200.ops import FtrlOptimizer
    FtrlOptimizer(0.01, l1_regularization_strength=0.5)
    with pytest.raises(NotImplementedError):
        FtrlOptimizer(0.01, learning_rate_power=-0.3)
    with pytest.raises(NotImplementedError):
        FtrlOptimizer(0.01, l2_shrinkage_regularization_strength=0.1)
    for kw in ({"l1_regularization_strength": -1.0}, {"l2_regularization_strength": -1.0},
               {"initial_accumulator_value": -0.1}, {"learning_rate_power": 0.5}):
        with pytest.raises(ValueError):
            FtrlOptimizer(0.01, **kw)
    with pytest.raises(ValueError):
        FtrlOptimizer(0.0)


def test_sparse_ftrl_equals_dense_ftrl_on_every_row():
    """Over several steps, TensorFlow's dense ApplyFtrl over the whole table leaves exactly what the row-sparse
    application to the touched rows leaves, L1 zeroing and L2 included."""
    rng = np.random.default_rng(5)
    R = 400
    for l1, l2 in ((0.5, 0.0), (0.0, 0.3), (0.02, 0.1)):
        dense = [np.zeros(R), np.zeros(R), np.full(R, 0.1)]
        sparse = [np.zeros(R), np.zeros(R), np.full(R, 0.1)]
        zeroed = 0
        for _ in range(6):
            rows = np.unique(rng.zipf(1.3, 120) % R)
            g = np.zeros(R)
            g[rows] = rng.normal(0, 1.0, rows.size)
            dense = list(W.ftrl_dense(*dense, g, 0.05, l1, l2))
            sparse = list(W.ftrl_rows(*sparse, g, rows, 0.05, l1, l2))
            for d, s in zip(dense, sparse):
                assert np.array_equal(d, s)
            zeroed += int(np.sum((dense[0] == 0) & (dense[1] != 0)))
        if l1 > 0.1:
            assert zeroed > 0          # L1 kept some touched rows at zero
        assert np.abs(dense[0]).max() > 0


def _ptr_arrays(n):
    return (C.c_int * max(n, 1))(), (C.c_void_p * max(n, 1))(), (C.c_void_p * max(n, 1))()


def test_c_abi_rejects_bad_wide_arguments():
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    bs, bi, bp = _ptr_arrays(0)
    base = 1 << 20          # never dereferenced: validation runs before any launch
    rc = lib.dr_wide_ftrl(base, 10, base, base, base, 4, 2, 0, bs, bi, bp, 0.0, 0.0, 0.0, None)
    assert rc == -1 and b"lr=" in lib.dr_last_error()
    assert lib.dr_wide_ftrl(base, 10, base, base, base, 4, 2, 0, bs, bi, bp, 0.1, -0.5, 0.0, None) == -1
    assert lib.dr_wide_ftrl(base, 10, base, base, base, 4, 2, 0, bs, bi, bp, 0.1, 0.0, -1.0, None) == -1
    rc = lib.dr_wide_ftrl(base + 4, 10, base, base, base, 4, 2, 0, bs, bi, bp, 0.1, 0.0, 0.0, None)
    assert rc == -1 and b"aligned" in lib.dr_last_error()
    for S in (0, 4097):
        assert lib.dr_wide_fwd(base, 10, base, base, base, 4, S, 0, bs, bi, bp, base, None) == -1
        assert lib.dr_wide_bwd(base, 10, base, base, base, 4, S, 0, bs, bi, bp, base, None) == -1
    assert lib.dr_wide_fwd(base, 10, base, base, base, 4, 2, 17, bs, bi, bp, base, None) == -1
    bs[0] = 2       # a bag slot outside [0, S)
    assert lib.dr_wide_fwd(base, 10, base, base, base, 4, 2, 1, bs, bi, bp, base, None) == -1
    vals = (C.c_void_p * 2)(base, base)
    none2 = (C.c_void_p * 2)()
    assert lib.dr_cross_hash_host(1, vals, none2, none2, 4, 0, 10, None, base) == -1
    assert lib.dr_cross_hash(2, vals, none2, none2, 4, 0, 0, None, base, None) == -1
    ragged = (C.c_void_p * 2)(base, None)
    rc = lib.dr_cross_hash(2, vals, none2, ragged, 4, 0, 10, None, base, None)
    assert rc == -1 and b"multi-valued" in lib.dr_last_error()


def test_c_abi_wide_rejections_in_order():
    """Every rejection of the three wide entries, with its code and exact text, in the order the checks run."""
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    base = 1 << 20          # never dereferenced: validation runs before any launch
    bs, bi, bp = _ptr_arrays(1)
    bi[0], bp[0] = base, base
    entries = {"dr_wide_fwd": lambda st, total, rows, B, S, n, slots, arg: lib.dr_wide_fwd(
                   st, total, rows, base, base, B, S, n, slots, bi, bp, arg, None),
               "dr_wide_bwd": lambda st, total, rows, B, S, n, slots, arg: lib.dr_wide_bwd(
                   st, total, rows, base, base, B, S, n, slots, bi, bp, arg, None),
               "dr_wide_ftrl": lambda st, total, rows, B, S, n, slots, arg: lib.dr_wide_ftrl(
                   st, total, rows, base, base, B, S, n, slots, bi, bp, arg, 0.0, 0.0, None)}
    first = {"dr_wide_fwd": "null logit", "dr_wide_bwd": "null g_logit",
             "dr_wide_ftrl": "lr=0 l1=0 l2=0 (need lr > 0, l1, l2 >= 0)"}
    for fn, call in entries.items():
        ok = 0.1 if fn == "dr_wide_ftrl" else base      # arg: the logit / g_logit pointer, or lr
        bad = 0.0 if fn == "dr_wide_ftrl" else None
        for args, msg in [
            ((base, 10, base, 4, 2, 0, bs, bad), first[fn]),
            ((base, 10, base, -1, 2, 0, bs, ok), "B=-1 S=2 total_rows=10"),
            ((base, 10, base, 4, 0, 0, bs, ok), "B=4 S=0 total_rows=10"),
            ((base, 10, base, 4, 4097, 17, bs, ok), "B=4 S=4097 total_rows=10"),
            ((base, -1, base, 4, 2, 0, bs, ok), "B=4 S=2 total_rows=-1"),
            ((None, 10, base, 4, 2, 17, bs, ok), "n_bags=17 (at most 16)"),
            ((base, 10, base, 4, 2, -1, bs, ok), "n_bags=-1 (at most 16)"),
            ((base, 10, None, 4, 2, 0, bs, ok), "null pointer"),
            ((base + 4, 10, base, 4, 2, 1, None, ok), "the state arena is not 16-B aligned"),
            ((base, 10, base, 4, 2, 1, None, ok), "null bag arrays"),
        ]:
            assert call(*args) == -1, (fn, args)
            assert lib.dr_last_error() == f"{fn}: {msg}".encode(), (fn, args)
        for slot in (2, -1):
            bs[0] = slot
            assert call(base, 10, base, 4, 2, 1, bs, ok) == -1
            assert lib.dr_last_error() == f"{fn}: bag 0: slot {slot} outside [0, 2) or null arrays".encode()
        bs[0] = 0


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="golden file not generated")
def test_oracle_matches_the_reference_model():
    """tests/golden/wdl_golden.npz comes from running the reference's wide_and_deep.py and dnn.py under the numpy
    TensorFlow stand-in; the float64 oracle must reproduce its output."""
    g = np.load(GOLDEN)
    n = int(g["n_cases"])
    assert n >= 1
    for k in range(n):
        p = f"c{k}_"
        B = int(g[p + "B"])
        S = int(g[p + "S"])
        wide_slots = []
        for s in range(int(g[p + "n_wide"])):
            ids, spl = g[f"{p}wide{s}_ids"], g[f"{p}wide{s}_splits"]
            wide_slots.append((int(g[f"{p}wide{s}_rows"]), int(g[f"{p}wide{s}_off"]),
                               [ids[spl[b]:spl[b + 1]].tolist() for b in range(B)]))
        look = W.wide_lookups(wide_slots, B)
        wide = W.wide_forward(g[p + "w"], float(g[p + "bias"]), look)
        deep_ids = [[[int(i)] for i in g[f"{p}deep{s}_ids"]] for s in range(S)]
        x = W.deep_embed([g[f"{p}table{s}"] for s in range(S)], deep_ids)
        L = int(g[p + "nlayers"])
        hs = W.tower_forward(x, [g[f"{p}k{i}"] for i in range(L)], [g[f"{p}b{i}"] for i in range(L)], "relu")
        prob = 1.0 / (1.0 + np.exp(-(wide + hs[-1][:, 0])))
        np.testing.assert_allclose(prob, g[p + "out"].reshape(-1), rtol=1e-10, atol=1e-12)
        # the golden's cross ids were made by the Python restatement (there is no TensorFlow crossing to run), so
        # this pins the library's host twin to the ids the golden model was evaluated with, not to TensorFlow
        from deep_recommenders_b200 import feature_column as fc
        from deep_recommenders_b200.hashing import cross_ids
        got = cross_ids(fc.crossed_column(["user_gender", "user_age"], 14),
                        {"user_gender": g[p + "gender"], "user_age": g[p + "age"]}, "cpu")
        assert got.tolist() == g[p + "cross_ids"].tolist()


def test_ftrl_accumulators_live_in_the_table():
    """The accumulator slot is initialised by the LinearTable, not by the optimizer's first apply, so a second
    optimizer continues from the trained slots; an optimizer whose initial_accumulator_value differs refuses."""
    import torch
    from deep_recommenders_b200.embedding import LinearTable
    from deep_recommenders_b200.ops import FtrlOptimizer
    t = LinearTable([3, 5], device="cpu")
    assert torch.equal(t.state[:, 2], torch.full((9,), 0.1))
    assert not t.state[:, [0, 1, 3]].any()
    t.lookups = (torch.zeros((1, 2), dtype=torch.int64), None)
    with pytest.raises(ValueError):
        FtrlOptimizer(0.01, initial_accumulator_value=0.2).apply(t)
    assert torch.equal(LinearTable([4], device="cpu", initial_accumulator_value=0.0).state[:, 2], torch.zeros(5))
    with pytest.raises(ValueError):
        LinearTable([4], device="cpu", initial_accumulator_value=-1.0)
