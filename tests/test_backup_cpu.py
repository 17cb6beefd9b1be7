"""Backup's checks that come before any device work (include/gamma_api.h, DESIGN.md §8): an engine without a path
refuses "create" with kInvalidArgument (4) and says why; "restore" (1) returns OK and writes nothing, as the
reference's BackupThread acts on "create" only.  Runs without a GPU."""
import ctypes as C
import os

import pytest

from vearch_b200 import _lib, engine


class CStatus(C.Structure):
    _fields_ = [("code", C.c_int), ("msg", C.c_void_p)]


def backup(h, command):
    l = _lib.lib()
    l.Backup.restype = CStatus
    l.Backup.argtypes = [C.c_void_p, C.c_int]
    st = l.Backup(h, command)
    msg = C.string_at(st.msg).decode() if st.msg else ""
    if st.msg:
        engine.libc.free(st.msg)
    return st.code, msg


@pytest.fixture
def eng(tmp_path):
    made = []

    def make(path):
        h = _lib.lib().gb_debug_engine_create(path.encode())
        assert h
        made.append(h)
        return h
    yield make
    for h in made:
        _lib.lib().Close.argtypes = [C.c_void_p]
        _lib.lib().Close(h)


def test_engine_without_path_is_refused(eng):
    code, msg = backup(eng(""), 0)
    assert code == 4 and "path" in msg


def test_restore_is_ok_and_writes_nothing(eng, tmp_path):
    h = eng(str(tmp_path / "p"))
    assert backup(h, 1) == (0, "")
    assert backup(eng(""), 1) == (0, "")
    assert not os.path.exists(tmp_path / "p")


def test_null_engine(eng):
    assert backup(None, 0)[0] == 4
