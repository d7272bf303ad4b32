"""The Adam entries of optim.cu and embed_adam.cu that the layer and sharded suites do not cover -- dr_adam_step,
dr_adam_advance[_hist], dr_lazy_adam_rows, dr_embed_adam_count, dr_embed_fm_bwd_adam[_tf], dr_embed_adam_prepare and
dr_embed_adam_flush -- reject bad arguments before any CUDA call, without a GPU.  Every call here is one the entry
refuses: an accepted one would launch a kernel on the fake address P."""
DR_EINVAL, DR_EALIGN = -1, -2
P = 1 << 12            # a 16-B aligned non-null address: never dereferenced, the checks fail first


def _lib():
    from deep_recommenders_b200 import _lib as L
    return L.load()


def _rejects(lib, rc, code, *needles):
    assert rc == code, rc
    msg = lib.dr_last_error()
    for n in needles:
        assert n.encode() in msg, msg


def test_adam_step_and_clocks():
    lib = _lib()
    step = lambda n=8, p=P, b1=0.9, b2=0.999, eps=1e-8: lib.dr_adam_step(p, P, P, P, n, 0.01, b1, b2, eps, 1, None,
                                                                        None)
    _rejects(lib, step(n=-1), DR_EINVAL, "dr_adam_step", "n=-1")
    _rejects(lib, step(p=None), DR_EINVAL, "dr_adam_step", "null pointer")
    _rejects(lib, step(b1=1.0), DR_EINVAL, "dr_adam_step", "out of range")
    _rejects(lib, step(b1=-0.5), DR_EINVAL, "dr_adam_step")
    _rejects(lib, step(b2=1.0), DR_EINVAL, "dr_adam_step")
    _rejects(lib, step(eps=-1e-8), DR_EINVAL, "dr_adam_step")
    adv = lambda s=P, lr_t=P, b1=0.9, b2=0.999: lib.dr_adam_advance(s, 0.01, b1, b2, lr_t, None)
    _rejects(lib, adv(s=None), DR_EINVAL, "dr_adam_advance", "null pointer")
    _rejects(lib, adv(lr_t=None), DR_EINVAL, "dr_adam_advance")
    _rejects(lib, adv(b1=1.0), DR_EINVAL, "dr_adam_advance", "out of range")
    _rejects(lib, adv(b2=-0.1), DR_EINVAL, "dr_adam_advance")
    hist = lambda s=P, b1=0.9, b2=0.999, n=16: lib.dr_adam_advance_hist(s, 0.01, b1, b2, P, P, n, None)
    _rejects(lib, hist(s=None), DR_EINVAL, "dr_adam_advance_hist", "null pointer")
    _rejects(lib, hist(b1=1.0), DR_EINVAL, "dr_adam_advance_hist", "out of range")
    _rejects(lib, hist(b2=1.5), DR_EINVAL, "dr_adam_advance_hist")
    _rejects(lib, hist(n=-1), DR_EINVAL, "dr_adam_advance_hist", "hist_len=-1")


def test_lazy_adam_rows():
    lib = _lib()
    call = lambda B=4, S=2, D=16, idb=8, ids=P, p=P, rs=32, flags=1, lp=None, lg=None, b1=0.9, eps=1e-8: \
        lib.dr_lazy_adam_rows(ids, idb, B, S, D, P, P, p, P, P, P, rs, flags, lp, lg, lg, lg, P, P, P, b1, 0.999, eps,
                              None)
    _rejects(lib, call(B=-1), DR_EINVAL, "dr_lazy_adam_rows", "B=-1")
    _rejects(lib, call(S=0), DR_EINVAL, "dr_lazy_adam_rows")
    _rejects(lib, call(S=4097), DR_EINVAL, "dr_lazy_adam_rows")
    _rejects(lib, call(D=6), DR_EINVAL, "dr_lazy_adam_rows", "D=6")
    _rejects(lib, call(D=132, rs=136), DR_EINVAL, "dr_lazy_adam_rows")
    _rejects(lib, call(idb=2), DR_EINVAL, "dr_lazy_adam_rows", "id_bytes=2")
    _rejects(lib, call(ids=None), DR_EINVAL, "dr_lazy_adam_rows", "null pointer")
    _rejects(lib, call(rs=16), DR_EINVAL, "dr_lazy_adam_rows", "row_stride=16")     # no room for the [w | pad] chunk
    _rejects(lib, call(flags=0, rs=18), DR_EINVAL, "dr_lazy_adam_rows")                # not a multiple of 4
    _rejects(lib, call(D=128, rs=132), DR_EINVAL, "dr_lazy_adam_rows")                 # [w | pad] needs D <= 124
    _rejects(lib, call(flags=0, rs=16, lp=P), DR_EINVAL, "dr_lazy_adam_rows", "lin_p given without")
    _rejects(lib, call(lp=P, lg=P), DR_EINVAL, "dr_lazy_adam_rows", "DR_EMBED_LIN_IN_ROW")
    _rejects(lib, call(p=P + 4), DR_EALIGN, "dr_lazy_adam_rows")
    _rejects(lib, call(b1=1.0), DR_EINVAL, "dr_lazy_adam_rows", "out of range")
    _rejects(lib, call(eps=-1.0), DR_EINVAL, "dr_lazy_adam_rows")


def test_embed_adam_count():
    lib = _lib()
    call = lambda B=4, S=2, D=16, idb=8, state=P: lib.dr_embed_adam_count(P, idb, B, S, D, P, P, state, None)
    _rejects(lib, call(B=-1), DR_EINVAL, "dr_embed_adam_count", "B=-1")
    _rejects(lib, call(S=0), DR_EINVAL, "dr_embed_adam_count")
    _rejects(lib, call(S=4097), DR_EINVAL, "dr_embed_adam_count")
    _rejects(lib, call(D=130), DR_EINVAL, "dr_embed_adam_count", "D=130")
    _rejects(lib, call(D=2), DR_EINVAL, "dr_embed_adam_count")
    _rejects(lib, call(idb=2), DR_EINVAL, "dr_embed_adam_count", "id_bytes=2")
    _rejects(lib, call(state=None), DR_EINVAL, "dr_embed_adam_count", "null pointer")


def _bwd(lib, tf, B=4, S=2, D=16, idb=8, ids=P, stack=P, sum_e=None, gl=P, gs=None, rs=32, ls=0, flags=1, state=P,
         lr_t=P, b1=0.9, b2=0.999, eps=1e-8, step=P, hist=P, hist_len=16):
    args = (ids, idb, P, P, stack, sum_e, gl, gs, B, S, D, rs, ls, flags, P, None, state, None)
    if tf:
        return lib.dr_embed_fm_bwd_adam_tf(*args, step, lr_t, hist, hist_len, 0.01, b1, b2, eps, None)
    return lib.dr_embed_fm_bwd_adam(*args, lr_t, b1, b2, eps, None)


def test_embed_fm_bwd_adam():
    lib = _lib()
    for tf, fn in ((False, "dr_embed_fm_bwd_adam"), (True, "dr_embed_fm_bwd_adam_tf")):
        call = lambda **kw: _bwd(lib, tf, **kw)
        _rejects(lib, call(B=-1), DR_EINVAL, fn, "B=-1")
        _rejects(lib, call(S=0), DR_EINVAL, fn)
        _rejects(lib, call(S=4097), DR_EINVAL, fn)
        _rejects(lib, call(D=6), DR_EINVAL, fn, "D=6")
        _rejects(lib, call(idb=2), DR_EINVAL, fn, "id_bytes=2")
        _rejects(lib, call(ids=None), DR_EINVAL, fn, "null pointer")
        _rejects(lib, call(lr_t=None), DR_EINVAL, fn, "null pointer")
        _rejects(lib, call(gl=None), DR_EINVAL, fn, "both g_logit and g_stack")
        _rejects(lib, call(stack=None), DR_EINVAL, fn, "stack is NULL")
        _rejects(lib, call(stack=P + 4), DR_EALIGN, fn)
        _rejects(lib, call(gs=P + 8), DR_EALIGN, fn)
        _rejects(lib, call(sum_e=P + 4), DR_EALIGN, fn)
        _rejects(lib, call(state=P + 4), DR_EALIGN, fn)
        _rejects(lib, call(rs=16), DR_EINVAL, fn, "bad strides")           # no room for the in-row weight
        _rejects(lib, call(flags=0, rs=18), DR_EINVAL, fn, "bad strides")  # not a multiple of 4
        _rejects(lib, call(flags=0, rs=16, ls=-1), DR_EINVAL, fn, "bad strides")
        _rejects(lib, call(b1=1.0), DR_EINVAL, fn, "out of range")
        _rejects(lib, call(b2=-0.1), DR_EINVAL, fn)
        _rejects(lib, call(eps=-1.0), DR_EINVAL, fn)
    _rejects(lib, _bwd(lib, True, step=None), DR_EINVAL, "dr_embed_fm_bwd_adam_tf", "step_dev is NULL")
    _rejects(lib, _bwd(lib, True, hist=None), DR_EINVAL, "dr_embed_fm_bwd_adam_tf", "bad lr history")
    _rejects(lib, _bwd(lib, True, hist_len=-1), DR_EINVAL, "dr_embed_fm_bwd_adam_tf", "bad lr history")


def test_embed_adam_prepare_and_flush():
    lib = _lib()
    prep = lambda B=4, S=2, D=16, idb=8, ids=P, tp=P, step=P: lib.dr_embed_adam_prepare(
        ids, idb, B, S, D, P, P, 32, 0, 1, tp, None, P, step, P, 16, 0.01, 0.9, 0.999, 1e-8, None)
    _rejects(lib, prep(B=-1), DR_EINVAL, "dr_embed_adam_prepare", "B=-1")
    _rejects(lib, prep(S=0), DR_EINVAL, "dr_embed_adam_prepare")
    _rejects(lib, prep(S=4097), DR_EINVAL, "dr_embed_adam_prepare")
    _rejects(lib, prep(D=132), DR_EINVAL, "dr_embed_adam_prepare", "D=132")
    _rejects(lib, prep(idb=2), DR_EINVAL, "dr_embed_adam_prepare", "id_bytes=2")
    _rejects(lib, prep(ids=None), DR_EINVAL, "dr_embed_adam_prepare", "null pointer")
    _rejects(lib, prep(tp=None), DR_EINVAL, "dr_embed_adam_prepare", "null pointer")
    _rejects(lib, prep(step=None), DR_EINVAL, "dr_embed_adam_prepare", "null pointer")
    flush = lambda S=2, D=16, total=12, state=P, step=P: lib.dr_embed_adam_flush(
        P, P, S, D, total, 32, 0, 1, P, None, state, step, P, 16, 0.01, 0.9, 0.999, 1e-8, None)
    _rejects(lib, flush(state=None), DR_EINVAL, "dr_embed_adam_flush", "null pointer")
    _rejects(lib, flush(step=None), DR_EINVAL, "dr_embed_adam_flush", "null pointer")
    _rejects(lib, flush(S=0), DR_EINVAL, "dr_embed_adam_flush", "S=0")
    _rejects(lib, flush(S=4097), DR_EINVAL, "dr_embed_adam_flush")
    _rejects(lib, flush(D=6), DR_EINVAL, "dr_embed_adam_flush", "D=6")
    _rejects(lib, flush(total=-1), DR_EINVAL, "dr_embed_adam_flush", "total_rows=-1")
