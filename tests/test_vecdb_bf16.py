"""gorse_b200_vecdb_storage: exported, and checks its collection before it needs a device; without a device no collection exists."""
import ctypes as C

import pytest


def test_storage_symbol_is_exported(gb):
    from gorse_b200 import _lib

    assert hasattr(_lib.lib, "gorse_b200_vecdb_storage")
    assert callable(gb.VectorCollection.storage)


def test_storage_of_null_collection_is_an_argument_error(gb):
    from gorse_b200 import _lib

    vb, nbytes = C.c_int32(-7), C.c_int64(-7)
    assert _lib.lib.gorse_b200_vecdb_storage(None, C.byref(vb), C.byref(nbytes)) == _lib.ERR_ARG
    assert b"NULL" in _lib.lib.gorse_b200_last_error()
    assert (vb.value, nbytes.value) == (-7, -7)   # nothing written
    assert _lib.lib.gorse_b200_vecdb_storage(None, None, None) == _lib.ERR_ARG


def test_no_collection_exists_without_a_device(gb):
    """The storage entry needs a collection, and a collection lives on a device: without one the context is refused, so no
    collection, and no storage answer, can exist."""
    try:
        have = gb.device_count() > 0
    except gb.GorseB200Error:   # no driver at all
        have = False
    if have:
        pytest.skip("a device is present")
    with pytest.raises(gb.GorseB200Error):
        gb.Context(0)
