"""CPU tests of search cancellation's host side: the cancel-token C-ABI and the kill registry behind SetKillStatus /
DeleteKillStatus (DESIGN.md section 8, cancellation).  No device is involved: without one a token is plain host memory,
which the registry sets exactly as it sets a running search's mapped word."""
from vearch_b200 import _lib
from vearch_b200 import index as gidx


def _kill(request_id, partition_id):
    _lib.lib().SetKillStatus(request_id.encode(), partition_id, 1)


def _unkill(request_id, partition_id):
    _lib.lib().DeleteKillStatus(request_id.encode(), partition_id)


def test_token_create_set_free():
    t = gidx.CancelToken()
    assert not t.is_set()
    t.set()
    assert t.is_set()
    t.set()  # setting twice leaves it set
    assert t.is_set()
    t.close()
    t.close()  # a closed token is freed once


def test_set_kill_sets_only_the_matching_pair():
    a, b, c = gidx.CancelToken(), gidx.CancelToken(), gidx.CancelToken()
    gidx.debug_cancel_register("cancel-cpu-1", 3, a)
    gidx.debug_cancel_register("cancel-cpu-1", 4, b)  # same request, other partition
    gidx.debug_cancel_register("cancel-cpu-2", 3, c)  # other request, same partition
    try:
        _kill("cancel-cpu-1", 3)
        assert a.is_set()
        assert not b.is_set() and not c.is_set()
        _kill("cancel-cpu-2", 3)
        assert c.is_set() and not b.is_set()
    finally:
        for rid, pid, t in (("cancel-cpu-1", 3, a), ("cancel-cpu-1", 4, b), ("cancel-cpu-2", 3, c)):
            gidx.debug_cancel_register(rid, pid, t, register=False)
            _unkill(rid, pid)


def test_registering_after_the_kill_sets_the_word():
    _kill("cancel-cpu-3", 0)
    t = gidx.CancelToken()
    try:
        gidx.debug_cancel_register("cancel-cpu-3", 0, t)
        assert t.is_set()
    finally:
        gidx.debug_cancel_register("cancel-cpu-3", 0, t, register=False)
        _unkill("cancel-cpu-3", 0)


def test_delete_kill_status_does_not_uncancel():
    t = gidx.CancelToken()
    gidx.debug_cancel_register("cancel-cpu-4", 1, t)
    try:
        _kill("cancel-cpu-4", 1)
        assert t.is_set()
        _unkill("cancel-cpu-4", 1)
        assert t.is_set()  # a running search stays cancelled
        u = gidx.CancelToken()
        gidx.debug_cancel_register("cancel-cpu-4", 1, u)  # the same request id is served again after the delete
        assert not u.is_set()
        gidx.debug_cancel_register("cancel-cpu-4", 1, u, register=False)
    finally:
        gidx.debug_cancel_register("cancel-cpu-4", 1, t, register=False)


def test_unregistered_token_is_left_alone():
    t = gidx.CancelToken()
    gidx.debug_cancel_register("cancel-cpu-5", 2, t)
    gidx.debug_cancel_register("cancel-cpu-5", 2, t, register=False)
    try:
        _kill("cancel-cpu-5", 2)
        assert not t.is_set()
    finally:
        _unkill("cancel-cpu-5", 2)
