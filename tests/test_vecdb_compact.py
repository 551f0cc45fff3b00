"""gorse_b200_vecdb_compact checks its collection before it needs a device."""
import ctypes as C


def test_compact_of_null_collection_is_an_argument_error(gb):
    from gorse_b200 import _lib

    new_slot, nbytes = (C.c_int64 * 4)(), (C.c_int64 * 2)()
    assert _lib.lib.gorse_b200_vecdb_compact(None, new_slot, nbytes) == _lib.ERR_ARG
    assert b"NULL" in _lib.lib.gorse_b200_last_error()
    assert _lib.lib.gorse_b200_vecdb_compact(None, None, None) == _lib.ERR_ARG
