"""The lookup entries -- the fused embedding gather / FM and its backward (plain and row-sharded), the TMA forward,
the bag lookups, FNN's input row, the row-sharded bucketing and permutation -- reject bad arguments before any CUDA
call, without a GPU, with the code and the exact dr_last_error() text below, checking in this order.  Every call here
is one the entry refuses: an accepted one would launch a kernel on the fake address P."""
import pytest

DR_EINVAL, DR_EALIGN, DR_ENOTSUP = -1, -2, -3
LIN_IN_ROW, NO_FM = 1, 2
P = 1 << 12            # a 16-B aligned non-null address: never dereferenced, the checks fail first


@pytest.fixture(scope="module")
def lib():
    from deep_recommenders_b200 import _lib as L
    return L.load()


def _check(lib, call, cases):
    for kw, code, msg in cases:
        assert call(**kw) == code, (kw, lib.dr_last_error())
        assert lib.dr_last_error() == msg.encode(), kw


def _dims(fn, d_join=" and"):
    """The shape and id-width checks every gather-shaped entry starts with; a call with two bad arguments reports the
    first in this order."""
    return [
        ({"B": -1}, DR_EINVAL, f"{fn}: B=-1 < 0"),
        ({"B": -1, "D": 6}, DR_EINVAL, f"{fn}: B=-1 < 0"),
        ({"S": 0}, DR_EINVAL, f"{fn}: S=0 outside [1,4096]"),
        ({"S": 4097, "id_bytes": 2}, DR_EINVAL, f"{fn}: S=4097 outside [1,4096]"),
        ({"D": 6}, DR_EINVAL, f"{fn}: D=6 unsupported (need D % 4 == 0{d_join} 4 <= D <= 128)"),
        ({"D": 0}, DR_EINVAL, f"{fn}: D=0 unsupported (need D % 4 == 0{d_join} 4 <= D <= 128)"),
        ({"D": 132, "id_bytes": 2}, DR_EINVAL, f"{fn}: D=132 unsupported (need D % 4 == 0{d_join} 4 <= D <= 128)"),
        ({"id_bytes": 2}, DR_EINVAL, f"{fn}: id_bytes=2 (need 4 or 8)"),
    ]


def test_embed_fm_fwd(lib):
    fn = "dr_embed_fm_fwd"

    def call(tab=P, rows=P, ids=P, id_bytes=8, B=4, S=2, D=16, rs=0, ls=0, flags=0, stack=P, sum_=P, logit=P):
        return lib.dr_embed_fm_fwd(tab, P, rows, ids, id_bytes, P, B, S, D, rs, ls, flags, stack, sum_, logit, None)

    _check(lib, call, _dims(fn) + [
        ({"tab": None}, DR_EINVAL, f"{fn}: null table_ptrs/rows/ids"),
        ({"rows": None}, DR_EINVAL, f"{fn}: null table_ptrs/rows/ids"),
        ({"ids": None, "stack": None, "sum_": None, "logit": None}, DR_EINVAL, f"{fn}: null table_ptrs/rows/ids"),
        ({"stack": None, "sum_": None, "logit": None}, DR_EINVAL, f"{fn}: no output requested"),
        ({"rs": 8}, DR_EINVAL, f"{fn}: row_stride=8 must be >= D and a multiple of 4"),
        ({"rs": 18, "ls": -1}, DR_EINVAL, f"{fn}: row_stride=18 must be >= D and a multiple of 4"),
        ({"ls": -1}, DR_EINVAL, f"{fn}: lin_stride=-1 < 1"),
        ({"flags": LIN_IN_ROW, "rs": 16}, DR_EINVAL, f"{fn}: DR_EMBED_LIN_IN_ROW needs row_stride >= D+4 and D <= 124"),
        ({"flags": LIN_IN_ROW, "D": 128, "rs": 132}, DR_EINVAL,
         f"{fn}: DR_EMBED_LIN_IN_ROW needs row_stride >= D+4 and D <= 124"),
        ({"stack": P + 4, "sum_": P + 4}, DR_EALIGN, f"{fn}: out_stack not 16-B aligned"),
        ({"sum_": P + 4}, DR_EALIGN, f"{fn}: out_sum not 16-B aligned"),
    ])


def test_embed_fm_bwd(lib):
    fn = "dr_embed_fm_bwd"

    def call(ids=P, id_bytes=8, rows=P, stack=P, sum_=P, gl=P, gs=P, B=4, S=2, D=16, rs=0, ls=0, flags=0, gt=P):
        return lib.dr_embed_fm_bwd(ids, id_bytes, rows, stack, sum_, gl, gs, B, S, D, rs, ls, flags, gt, P, P, 1.0,
                                   None)

    _check(lib, call, _dims(fn) + [
        ({"ids": None}, DR_EINVAL, f"{fn}: null ids/rows/grad_table_ptrs"),
        ({"gt": None, "gl": None, "gs": None}, DR_EINVAL, f"{fn}: null ids/rows/grad_table_ptrs"),
        ({"gl": None, "gs": None}, DR_EINVAL, f"{fn}: both g_logit and g_stack are NULL"),
        ({"stack": None}, DR_EINVAL, f"{fn}: g_logit given but stack is NULL"),
        ({"stack": P + 4, "gs": P + 4}, DR_EALIGN, f"{fn}: stack not 16-B aligned"),
        ({"gs": P + 8}, DR_EALIGN, f"{fn}: g_stack not 16-B aligned"),
        ({"sum_": P + 4, "rs": 8}, DR_EALIGN, f"{fn}: sum_e not 16-B aligned"),
        ({"rs": 8}, DR_EINVAL, f"{fn}: bad strides row=8 lin=1"),
        ({"ls": -2}, DR_EINVAL, f"{fn}: bad strides row=16 lin=-2"),
        ({"flags": LIN_IN_ROW, "rs": 16}, DR_EINVAL, f"{fn}: DR_EMBED_LIN_IN_ROW needs row_stride >= D+4 and D <= 124"),
    ])


def test_embed_fm_fwd_sharded(lib):
    fn = "dr_embed_fm_fwd_sharded"

    def call(peers=P, world=2, id_bytes=8, B=4, S=2, D=16, rs=20, flags=LIN_IN_ROW, lin_off=0, stack=P, logit=P):
        return lib.dr_embed_fm_fwd_sharded(peers, world, P, P, P, id_bytes, P, B, S, D, rs, flags, lin_off, stack,
                                           None, logit, None)

    _check(lib, call, _dims(fn) + [
        ({"flags": NO_FM}, DR_ENOTSUP, f"{fn}: DR_EMBED_NO_FM is not served"),
        ({"flags": NO_FM, "B": 0}, DR_ENOTSUP, f"{fn}: DR_EMBED_NO_FM is not served"),
        ({"lin_off": -1}, DR_EINVAL, f"{fn}: lin_offset=-1 (must be >= 0 and exclusive with DR_EMBED_LIN_IN_ROW)"),
        ({"lin_off": 64}, DR_EINVAL, f"{fn}: lin_offset=64 (must be >= 0 and exclusive with DR_EMBED_LIN_IN_ROW)"),
        ({"peers": None}, DR_EINVAL, f"{fn}: null pointer"),
        ({"world": 0}, DR_EINVAL, f"{fn}: world=0 outside [1,64]"),
        ({"world": 65}, DR_EINVAL, f"{fn}: world=65 outside [1,64]"),
        ({"stack": None, "logit": None}, DR_EINVAL, f"{fn}: no output requested"),
        ({"rs": 16}, DR_EINVAL, f"{fn}: bad row_stride=16 for D=16"),
        ({"flags": 0, "rs": 12}, DR_EINVAL, f"{fn}: bad row_stride=12 for D=16"),
        ({"D": 128, "rs": 132}, DR_EINVAL, f"{fn}: bad row_stride=132 for D=128"),
        ({"stack": P + 4}, DR_EALIGN, f"{fn}: out_stack not 16-B aligned"),
    ])


def test_embed_fm_bwd_sharded(lib):
    fn = "dr_embed_fm_bwd_sharded"

    def call(peers=P, world=2, id_bytes=8, stack=P, gl=P, gs=P, B=4, S=2, D=16, rs=20, flags=LIN_IN_ROW, lin_off=0):
        return lib.dr_embed_fm_bwd_sharded(peers, world, P, P, P, id_bytes, stack, P, gl, gs, B, S, D, rs, flags,
                                           lin_off, P, 1.0, None)

    _check(lib, call, _dims(fn) + [
        ({"flags": NO_FM}, DR_ENOTSUP, f"{fn}: DR_EMBED_NO_FM is not served"),
        ({"lin_off": -1}, DR_EINVAL, f"{fn}: lin_offset=-1 (must be >= 0 and exclusive with DR_EMBED_LIN_IN_ROW)"),
        ({"lin_off": 64}, DR_EINVAL, f"{fn}: lin_offset=64 (must be >= 0 and exclusive with DR_EMBED_LIN_IN_ROW)"),
        ({"peers": None}, DR_EINVAL, f"{fn}: null pointer"),
        ({"world": 0}, DR_EINVAL, f"{fn}: world=0 outside [1,64]"),
        ({"world": 65, "gl": None, "gs": None}, DR_EINVAL, f"{fn}: world=65 outside [1,64]"),
        ({"gl": None, "gs": None}, DR_EINVAL, f"{fn}: both g_logit and g_stack are NULL"),
        ({"stack": None}, DR_EINVAL, f"{fn}: g_logit given but stack is NULL"),
        ({"rs": 16}, DR_EINVAL, f"{fn}: bad row_stride=16 for D=16"),
        ({"flags": 0, "rs": 18}, DR_EINVAL, f"{fn}: bad row_stride=18 for D=16"),
    ])


def test_embed_fm_fwd_tma(lib):
    fn = "dr_embed_fm_fwd_tma"

    def call(arena=P, total=100, id_bytes=8, B=4, S=4, D=16, rs=32, stack=P, sum_=P):
        return lib.dr_embed_fm_fwd_tma(arena, total, P, P, P, id_bytes, P, B, S, D, rs, stack, sum_, P, None)

    served = "this variant serves fused rows with D=16, S<=32"
    _check(lib, call, [
        ({"arena": None, "B": -1}, DR_EINVAL, f"{fn}: null pointer"),
        ({"B": -1}, DR_EINVAL, f"{fn}: B=-1 S=4"),
        ({"S": 0, "id_bytes": 2}, DR_EINVAL, f"{fn}: B=4 S=0"),
        ({"id_bytes": 2, "D": 8}, DR_EINVAL, f"{fn}: id_bytes=2 (need 4 or 8)"),
        ({"D": 32}, DR_ENOTSUP, f"{fn}: {served} (got D=32 S=4 stride=32)"),
        ({"S": 33}, DR_ENOTSUP, f"{fn}: {served} (got D=16 S=33 stride=32)"),
        ({"rs": 16}, DR_ENOTSUP, f"{fn}: {served} (got D=16 S=4 stride=16)"),
        ({"rs": 22}, DR_ENOTSUP, f"{fn}: {served} (got D=16 S=4 stride=22)"),
        ({"total": 0}, DR_ENOTSUP, f"{fn}: {served} (got D=16 S=4 stride=32)"),
        ({"total": (1 << 31) - 1}, DR_ENOTSUP, f"{fn}: {served} (got D=16 S=4 stride=32)"),
        ({"arena": P + 4}, DR_EALIGN, f"{fn}: arena / out_stack / out_sum not 16-B aligned"),
        ({"stack": P + 4}, DR_EALIGN, f"{fn}: arena / out_stack / out_sum not 16-B aligned"),
        ({"sum_": P + 8}, DR_EALIGN, f"{fn}: arena / out_stack / out_sum not 16-B aligned"),
    ])


def _gather_cases(fn, bases):
    return [(kw, code, msg) for kw, code, msg in _dims(fn) if "S" not in kw] + [
        ({"tab": None}, DR_EINVAL, f"{fn}: null pointer"),
        ({"ids": None, "rows": -1}, DR_EINVAL, f"{fn}: null pointer"),
        ({"x": None}, DR_EINVAL, f"{fn}: null pointer"),
        ({"rows": -1, "tab": P + 4}, DR_EINVAL, f"{fn}: rows < 0"),
        ({"tab": P + 4}, DR_EALIGN, f"{fn}: {bases} not 16-B aligned"),
        ({"x": P + 8}, DR_EALIGN, f"{fn}: {bases} not 16-B aligned"),
    ]


def test_gather_and_scatter_add(lib):
    def gather(tab=P, rows=10, ids=P, id_bytes=8, B=4, D=16, x=P):
        return lib.dr_gather_fwd(tab, rows, ids, id_bytes, B, D, x, None)

    def scatter(tab=P, rows=10, ids=P, id_bytes=8, B=4, D=16, x=P):
        return lib.dr_scatter_add(tab, rows, ids, id_bytes, B, D, x, 1.0, None)

    _check(lib, gather, _gather_cases("dr_gather_fwd", "table/out"))
    _check(lib, scatter, _gather_cases("dr_scatter_add", "table/g"))


def test_embed_bag(lib):
    def fwd(ids=P, id_bytes=8, splits=P, B=4, D=16, comb=1, rows=10, rs=16, x=P, t=P, xs=16):
        return lib.dr_embed_bag_fwd(t, rows, rs, ids, id_bytes, splits, B, D, comb, x, xs, None)

    def bwd(ids=P, id_bytes=8, splits=P, B=4, D=16, comb=1, rows=10, rs=16, x=P, t=P, xs=16):
        return lib.dr_embed_bag_bwd(ids, id_bytes, splits, B, D, comb, x, xs, rows, rs, t, 1.0, None)

    for call, fn, nulls, stride in ((fwd, "dr_embed_bag_fwd", "null table / out", "out_stride"),
                                    (bwd, "dr_embed_bag_bwd", "null g_out / grad_table", "g_stride")):
        _check(lib, call, [
            ({"B": -1, "D": 0}, DR_EINVAL, f"{fn}: B=-1 < 0"),
            ({"D": 0}, DR_EINVAL, f"{fn}: D=0 outside [1,1024]"),
            ({"D": 1025, "rows": 0}, DR_EINVAL, f"{fn}: D=1025 outside [1,1024]"),
            ({"rows": 0}, DR_EINVAL, f"{fn}: rows=0 row_stride=16 (need >= D=16)"),
            ({"rs": 8, "id_bytes": 2}, DR_EINVAL, f"{fn}: rows=10 row_stride=8 (need >= D=16)"),
            ({"id_bytes": 2}, DR_EINVAL, f"{fn}: id_bytes=2 (need 4 or 8)"),
            ({"comb": 3, "splits": None}, DR_EINVAL, f"{fn}: combiner=3"),
            ({"comb": -1}, DR_EINVAL, f"{fn}: combiner=-1"),
            ({"splits": None}, DR_EINVAL, f"{fn}: null ids / row_splits"),
            ({"ids": None, "t": None}, DR_EINVAL, f"{fn}: null ids / row_splits"),
            ({"t": None}, DR_EINVAL, f"{fn}: {nulls}"),
            ({"x": None, "xs": 8}, DR_EINVAL, f"{fn}: {nulls}"),
            ({"xs": 8}, DR_EINVAL, f"{fn}: {stride}=8 < D=16"),
        ])


def test_fnn_input(lib):
    S, D = 3, 16
    ld = 4 + S * D          # P = round_up(1 + S, 4) = 4

    def fwd(tab=P, lin=P, rows=P, ids=P, id_bytes=8, rs=20, ls=0, flags=LIN_IN_ROW, bias=P, B=4, S=S, D=D, ld=ld, x=P):
        return lib.dr_fnn_input_fwd(tab, lin, rows, ids, id_bytes, rs, ls, flags, bias, B, S, D, ld, x, None)

    def bwd(tab=P, lin=P, rows=P, ids=P, id_bytes=8, rs=20, ls=0, flags=LIN_IN_ROW, bias=P, B=4, S=S, D=D, ld=ld, x=P):
        return lib.dr_fnn_input_bwd(ids, id_bytes, rows, x, B, S, D, ld, rs, ls, flags, tab, lin, 1.0, None)

    for call, fn in ((fwd, "dr_fnn_input_fwd"), (bwd, "dr_fnn_input_bwd")):
        nulls = f"{fn}: null table pointers / rows / ids / row buffer"
        _check(lib, call, [
            ({"tab": None, "B": -1}, DR_EINVAL, nulls),
            ({"rows": None}, DR_EINVAL, nulls),
            ({"ids": None}, DR_EINVAL, nulls),
            ({"x": None}, DR_EINVAL, nulls),
        ] + _dims(fn, ",") + [
            ({"ld": ld - 1}, DR_EINVAL, f"{fn}: ld={ld - 1}, the row layout needs P + S*D = {ld}"),
            ({"S": 4, "ld": ld}, DR_EINVAL, f"{fn}: ld={ld}, the row layout needs P + S*D = 72"),
            ({"flags": NO_FM}, DR_EINVAL, f"{fn}: flags=2 (only DR_EMBED_LIN_IN_ROW)"),
            ({"flags": 0, "rs": 8}, DR_EINVAL, f"{fn}: row_stride=8 must be >= D and a multiple of 4"),
            ({"rs": 18}, DR_EINVAL, f"{fn}: row_stride=18 must be >= D and a multiple of 4"),
            ({"rs": 16}, DR_EINVAL, f"{fn}: DR_EMBED_LIN_IN_ROW needs row_stride >= D+4 and D <= 124"),
            ({"flags": 0, "rs": 16, "lin": None}, DR_EINVAL, f"{fn}: the split layout needs lin_ptrs and lin_stride >= 1"),
            ({"flags": 0, "rs": 16, "ls": -1}, DR_EINVAL, f"{fn}: the split layout needs lin_ptrs and lin_stride >= 1"),
            ({"x": P + 4, "B": 1 << 30}, DR_EALIGN, f"{fn}: the [B, ld] row buffer is not 16-B aligned"),
            ({"B": 1 << 30, "S": 2, "ld": 36}, DR_ENOTSUP, f"{fn}: B*S=2147483648 >= 2^31 lookups"),
        ])
    _check(lib, fwd, [({"bias": None}, DR_EINVAL, "dr_fnn_input_fwd: null bias")])


def test_shard_bucket_ids(lib):
    fn = "dr_shard_bucket_ids"

    def call(ids=P, id_bytes=8, n=8, S=2, G=2, cap=16, counts=P):
        return lib.dr_shard_bucket_ids(ids, id_bytes, n, S, P, P, G, cap, counts, P, P, P, None)

    _check(lib, call, [
        ({"ids": None, "n": -1}, DR_EINVAL, f"{fn}: null pointer"),
        ({"counts": None}, DR_EINVAL, f"{fn}: null pointer"),
        ({"n": -1, "G": 0}, DR_EINVAL, f"{fn}: n=-1 < 0"),
        ({"G": 0}, DR_EINVAL, f"{fn}: G=0 outside [1,64]"),
        ({"G": 65, "S": 0}, DR_EINVAL, f"{fn}: G=65 outside [1,64]"),
        ({"S": 0, "cap": 0}, DR_EINVAL, f"{fn}: S=0"),
        ({"cap": 0}, DR_EINVAL, f"{fn}: G*cap=0 must fit int32"),
        ({"cap": 1 << 30, "id_bytes": 2}, DR_EINVAL, f"{fn}: G*cap=2147483648 must fit int32"),
        ({"id_bytes": 2}, DR_EINVAL, f"{fn}: id_bytes=2"),
    ])


@pytest.mark.parametrize("entry", ["dr_permute_rows", "dr_unpermute_rows"])
def test_permute_rows(lib, entry):
    fn = "dr_permute_rows"          # both directions report under the name of the forward entry

    def call(x=P, perm=P, n=8, D=16, out=P):
        return getattr(lib, entry)(x, perm, n, D, out, None)

    _check(lib, call, [
        ({"x": None, "n": -1}, DR_EINVAL, f"{fn}: null pointer"),
        ({"perm": None}, DR_EINVAL, f"{fn}: null pointer"),
        ({"n": -1, "x": P + 4}, DR_EINVAL, f"{fn}: bad shape n=-1 D=16"),
        ({"D": 6}, DR_EINVAL, f"{fn}: bad shape n=8 D=6"),
        ({"D": 0}, DR_EINVAL, f"{fn}: bad shape n=8 D=0"),
        ({"x": P + 4}, DR_EALIGN, f"{fn}: in/out not 16-B aligned"),
        ({"out": P + 8}, DR_EALIGN, f"{fn}: in/out not 16-B aligned"),
    ])
