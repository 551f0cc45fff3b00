"""gorse_b200_fm_fit_trials' argument checks, which run on the host before the device is touched (the context last): with a
NULL context every bad argument is still reported, so no GPU is needed."""
import ctypes as C

import numpy as np
import pytest

import fm_oracle


def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def call(_lib, nf=40, k=8, trials=None, n_trials=None, pins=None, n_params=None, rows=None, dims=(), mask=None):
    rng = np.random.default_rng(3)
    tr, te = fm_oracle.random_ctr(rng, nf, 60), fm_oracle.random_ctr(rng, nf, 20)
    if trials is None:
        trials = [dict(), dict(lr=0.02)]
    fps = (_lib.FMFitParams * len(trials))()
    for i, over in enumerate(trials):
        fps[i] = _lib.FMFitParams(k, 2, 0.01, 0.0, 0, 16, 1, 0, 0)
        for key, v in over.items():
            setattr(fps[i], key, v)
    want = 1 + nf * k + nf + sum(k * (3 * d + 2) for d in dims)
    if pins is None:
        pins = [np.zeros(want, np.float32) for _ in trials]
    pin_arr = (C.c_void_p * len(pins))(*[None if p is None else p.ctypes.data for p in pins])
    tabs = [np.zeros((5, d), np.uint16) for d in dims]
    tab_arr = (C.c_void_p * max(len(tabs), 1))(*[t.ctypes.data for t in tabs])
    dim_arr = np.array(dims, np.int32)
    if rows is None:
        rows = (np.zeros(60, np.int32), np.zeros(20, np.int32))
    res = (_lib.FMFitResult * len(trials))()
    return _lib.lib.gorse_b200_fm_fit_trials(
        None, nf, 4, len(trials) if n_trials is None else n_trials, C.cast(fps, C.c_void_p),
        60, ptr(tr[0]), ptr(tr[1]), ptr(tr[2]), ptr(tr[3]), ptr(rows[0]) if dims else None,
        20, ptr(te[0]), ptr(te[1]), ptr(te[2]), ptr(te[3]), ptr(rows[1]) if dims else None,
        len(dims), ptr(dim_arr) if dims else None, 5, tab_arr if dims else None, ptr(mask),
        C.cast(pin_arr, C.c_void_p), want if n_params is None else n_params, None, None, None, None, C.cast(res, C.c_void_p))


@pytest.mark.parametrize("field,value", [("n_factors", 4), ("batch_size", 8), ("verbose", 2), ("patience", 3), ("max_steps", 5)])
def test_unequal_shared_fields(gb, field, value):
    from gorse_b200 import _lib

    pins = None
    if field == "n_factors":   # trial 1's own model size, so only the sharing rule is broken
        pins = [np.zeros(1 + 40 * 8 + 40, np.float32), np.zeros(1 + 40 * 4 + 40, np.float32)]
    assert call(_lib, trials=[dict(), {field: value}], pins=pins) == _lib.ERR_ARG
    assert b"trial 1" in _lib.lib.gorse_b200_last_error()


def test_fields_that_may_differ_pass_the_checks(gb):
    from gorse_b200 import _lib

    # lr, reg, optimizer and n_epochs differ: every check passes and only the NULL context is left
    assert call(_lib, trials=[dict(), dict(lr=0.5, reg=0.1, optimizer=1, n_epochs=7)]) == _lib.ERR_ARG
    assert b"ctx" in _lib.lib.gorse_b200_last_error()


@pytest.mark.parametrize("n", [0, -1])
def test_no_trials(gb, n):
    from gorse_b200 import _lib

    assert call(_lib, n_trials=n) == _lib.ERR_ARG


def test_null_params_in(gb):
    from gorse_b200 import _lib

    assert call(_lib, pins=[np.zeros(1 + 40 * 8 + 40, np.float32), None]) == _lib.ERR_ARG
    assert b"params_in[1]" in _lib.lib.gorse_b200_last_error()


@pytest.mark.parametrize("delta", [-1, 1])
def test_wrong_n_params(gb, delta):
    from gorse_b200 import _lib

    assert call(_lib, n_params=1 + 40 * 8 + 40 + delta) == _lib.ERR_ARG
    assert b"n_params" in _lib.lib.gorse_b200_last_error()


@pytest.mark.parametrize("bad", [5, -2])
def test_out_of_range_table_rows(gb, bad):
    from gorse_b200 import _lib

    tr_rows = np.zeros(60, np.int32)
    tr_rows[7] = bad
    assert call(_lib, dims=(6,), rows=(tr_rows, np.zeros(20, np.int32))) == _lib.ERR_ARG
    assert b"table row" in _lib.lib.gorse_b200_last_error()
    te_rows = np.zeros(20, np.int32)
    te_rows[3] = bad
    assert call(_lib, dims=(6,), rows=(np.zeros(60, np.int32), te_rows)) == _lib.ERR_ARG


def test_unsupported_shapes(gb):
    from gorse_b200 import _lib

    assert call(_lib, k=33) == _lib.ERR_UNSUPPORTED
    assert call(_lib, dims=(1025,)) == _lib.ERR_UNSUPPORTED
    assert call(_lib, dims=(2,) * 9) == _lib.ERR_UNSUPPORTED


def test_bad_trial_params(gb):
    from gorse_b200 import _lib

    assert call(_lib, trials=[dict(), dict(optimizer=2)]) == _lib.ERR_ARG
    assert call(_lib, trials=[dict(), dict(n_epochs=-1)]) == _lib.ERR_ARG
