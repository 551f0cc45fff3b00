"""gorse_b200_cf_fit_trials checks its arguments on the host before it touches the device: every error below is
reported without a CUDA device (the model is checked last, so a NULL one reaches the other checks first)."""
import ctypes as C

import numpy as np
import pytest


def call(_lib, trials, als=None, results=True, n=None):
    k = len(trials)
    fps = (_lib.FitParams * max(k, 1))(*trials)
    res = (_lib.FitResult * max(k, 1))() if results else None
    als = np.zeros(max(k, 1), np.int32) if als is None else np.asarray(als, np.int32)
    toff = np.zeros(2, np.int64)
    st = _lib.lib.gorse_b200_cf_fit_trials(None, k if n is None else n, als.ctypes.data_as(C.c_void_p), C.cast(fps, C.c_void_p),
                                           toff.ctypes.data_as(C.c_void_p), None, None, None, None, None,
                                           C.cast(res, C.c_void_p) if results else None, None, None)
    return st, _lib.lib.gorse_b200_last_error().decode()


def params(_lib, als=0, **kw):
    p = _lib.FitParams()
    assert _lib.lib.gorse_b200_fit_params_default(als, C.byref(p)) == _lib.OK
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.fixture
def lib(gb):
    from gorse_b200 import _lib

    return _lib


def test_null_model(lib):
    st, msg = call(lib, [params(lib), params(lib, lr=0.01)])
    assert st == lib.ERR_ARG and "cf is NULL" in msg


def test_no_trials(lib):
    st, msg = call(lib, [params(lib)], n=0)
    assert st == lib.ERR_ARG and "n_trials" in msg


@pytest.mark.parametrize("field,value", [("seed", 5), ("verbose", 3), ("n_factors", 32), ("candidates", 50), ("topk", 5),
                                         ("patience", 2)])
def test_shared_fields_must_match(lib, field, value):
    st, msg = call(lib, [params(lib), params(lib, lr=0.02, **{field: value})])
    assert st == lib.ERR_ARG and "trial 1" in msg and "must equal" in msg


def test_per_trial_fields_may_differ(lib):
    # lr, reg, init_stddev, alpha, n_epochs and the kind differ: only the model is missing
    st, msg = call(lib, [params(lib, lr=0.01, n_epochs=5), params(lib, 1, reg=0.5, alpha=0.2, init_stddev=0.3, n_epochs=7)], als=[0, 1])
    assert st == lib.ERR_ARG and "cf is NULL" in msg


def test_null_results(lib):
    st, msg = call(lib, [params(lib)], results=False)
    assert st == lib.ERR_ARG and "NULL" in msg


def test_each_trial_is_checked_like_a_solo_fit(lib):
    st, msg = call(lib, [params(lib), params(lib, n_epochs=-1)])
    assert st == lib.ERR_ARG and "n_epochs" in msg
    st, msg = call(lib, [params(lib, topk=0), params(lib, topk=0)])
    assert st == lib.ERR_ARG and "topk" in msg
