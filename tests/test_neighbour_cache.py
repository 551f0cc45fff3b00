"""gorse_b200_vecdb_neighbour_cache / _stats: exported, and every argument check that needs no collection answers before the
collection is read.  Without a device no collection exists, so nothing here is answered on the host."""
import ctypes as C

import pytest


def test_symbols_exist(gb):
    from gorse_b200 import _lib

    assert hasattr(_lib.lib, "gorse_b200_vecdb_neighbour_cache")
    assert hasattr(_lib.lib, "gorse_b200_vecdb_neighbour_cache_stats")
    assert hasattr(gb.VectorCollection, "neighbour_cache") and hasattr(gb.VectorCollection, "neighbour_cache_stats")


def test_null_collection_and_stats_are_argument_errors(gb):
    from gorse_b200 import _lib

    lib = _lib.lib
    assert lib.gorse_b200_vecdb_neighbour_cache(None, 10, 100) == _lib.ERR_ARG
    assert b"NULL" in lib.gorse_b200_last_error()
    assert lib.gorse_b200_vecdb_neighbour_cache(None, 10, 0) == _lib.ERR_ARG
    stats = (C.c_int64 * 7)(*([-5] * 7))
    assert lib.gorse_b200_vecdb_neighbour_cache_stats(None, stats) == _lib.ERR_ARG
    assert list(stats) == [-5] * 7, "a refused call writes nothing"
    assert lib.gorse_b200_vecdb_neighbour_cache_stats(None, None) == _lib.ERR_ARG


@pytest.mark.parametrize("n, rows, word", [(0, 10, b"n = 0"), (-1, 10, b"n = -1"), (1025, 10, b"n = 1025"), (10, -1, b"negative rows"),
                                           (0, -1, b"negative rows")])
def test_out_of_range_arguments_are_refused_before_the_collection(gb, n, rows, word):
    """n outside [1, 1024] and negative rows are ERR_ARG whatever the collection (the sparse limit of 128 and Cosine need one:
    GORSE_B200_ERR_UNSUPPORTED, checked on the GPU)"""
    from gorse_b200 import _lib

    assert _lib.lib.gorse_b200_vecdb_neighbour_cache(None, n, rows) == _lib.ERR_ARG
    assert word in _lib.lib.gorse_b200_last_error()


def test_without_a_device_no_collection_is_made(gb):
    """the cache belongs to a collection, and a collection needs a device: without one, nothing is answered on the host"""
    from gorse_b200 import _lib

    cnt = C.c_int32(-1)
    if _lib.lib.gorse_b200_device_count(C.byref(cnt)) == _lib.OK and cnt.value > 0:
        pytest.skip("a device is present")
    with pytest.raises(gb.GorseB200Error):
        gb.Context(0)
