"""gorse_b200_vecdb_neighbour_cache_fill / _save / _load: exported, bound in Python, called by the Go store, and every NULL
argument is refused before a collection is read.  Without a device no collection exists, so nothing more is answered here."""
import ctypes as C
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("gorse_b200_vecdb_neighbour_cache_fill", "gorse_b200_vecdb_neighbour_cache_save", "gorse_b200_vecdb_neighbour_cache_load")


def test_symbols_exist(gb):
    from gorse_b200 import _lib

    for name in ENTRIES:
        assert hasattr(_lib.lib, name), name
    for m in ("neighbour_cache_fill", "save_neighbour_cache", "load_neighbour_cache"):
        assert hasattr(gb.VectorCollection, m), m


def test_null_arguments_are_refused(gb):
    from gorse_b200 import _lib

    lib = _lib.lib
    stats = (C.c_int64 * 4)(*([-5] * 4))
    assert lib.gorse_b200_vecdb_neighbour_cache_fill(None, stats) == _lib.ERR_ARG
    assert b"NULL" in lib.gorse_b200_last_error()
    assert list(stats) == [-5] * 4, "a refused call writes nothing"
    assert lib.gorse_b200_vecdb_neighbour_cache_fill(None, None) == _lib.ERR_ARG
    write = _lib.WRITE_FN(lambda user, buf, n: 0)
    read = _lib.READ_FN(lambda user, buf, n: 0)
    nbytes = C.c_int64(-5)
    assert lib.gorse_b200_vecdb_neighbour_cache_save(None, write, None, C.byref(nbytes)) == _lib.ERR_ARG
    assert lib.gorse_b200_vecdb_neighbour_cache_save(None, None, None, None) == _lib.ERR_ARG
    assert nbytes.value == -5
    st3 = (C.c_int64 * 3)(*([-5] * 3))
    assert lib.gorse_b200_vecdb_neighbour_cache_load(None, read, None, st3) == _lib.ERR_ARG
    assert lib.gorse_b200_vecdb_neighbour_cache_load(None, None, None, None) == _lib.ERR_ARG
    assert list(st3) == [-5] * 3


def test_header_documents_the_stream():
    src = open(os.path.join(ROOT, "include", "gorse_b200.h")).read()
    assert '"GB200NBR"' in src and "Neighbour stream format, version 1" in src
    for name in ENTRIES:
        assert re.search(r"int32_t %s\(" % name, src), name


def test_go_store_calls_the_new_entries():
    """the writing process fills and saves, a reading process loads (the shim is not compiled here; tests/test_abi.py checks
    that every call it names is declared)"""
    go = open(os.path.join(ROOT, "go", "storage", "vectors", "b200.go")).read()
    for name in ENTRIES:
        assert "C.%s(" % name in go, name
    assert "neighbour_fill_n" in go


def test_go_writer_puts_the_lists_in_place_before_the_collection_file():
    """a reader that reloads a new collection file must find that generation's lists already there: save() writes
    <file>.nbr before it renames the collection file into place"""
    go = open(os.path.join(ROOT, "go", "storage", "vectors", "b200.go")).read()
    body = go[go.index("func (db *B200) save(name string, c *b200Collection) error {"):]
    body = body[:body.index("\n}\n")]
    assert body.index("db.saveNeighbours(name, c, generation)") < body.index('os.Rename(path+".tmp", path)')
