"""libbkgpu.so driven from several host threads at once, on the CPU: plan lowering (bkgpu_plan_explain) and the calling thread's error
text (bkgpu_last_error(NULL)).  A store lowers one plan per request on many threads; every answer must be the one a single thread gets,
and each thread must read its own last message, never another thread's.  ctypes releases the GIL for the duration of each call, so the
calls overlap inside the library."""
import ctypes
import random
import threading

import pytest

from baikaldb_b200 import _lib, queries
from baikaldb_b200 import plan as P
from baikaldb_b200.plan import PrimitiveType as T
from tests import fuzz_plans

THREADS = 8
ROUNDS = 6
TEXT_LEN = 1 << 16


def _descriptors():
    """(name, plan bytes): valid plans of every kind, and malformed or refused ones whose messages differ from each other"""
    out = [("c1", queries.c1_count_where().serialize()), ("c2", queries.c2_filter_groupby().serialize()),
           ("c2_merge", queries.c2_filter_groupby(merge=True).serialize()), ("c3", queries.c3_join_groupby().serialize()),
           ("c5", queries.c5_topk().serialize()), ("c5_desc", queries.c5_topk(77, asc=False).serialize()),
           ("c6", queries.c6_star_groupby().serialize()), ("c6_window", queries.c6_star_window().serialize())]
    out += [(f"fuzz{s}", fuzz_plans.fragment(s)[0].serialize()) for s in range(12)]
    c2 = queries.c2_filter_groupby().serialize()
    out += [(f"truncated{n}", c2[:n]) for n in (0, 4, 12, 40, len(c2) // 2, len(c2) - 4)]
    out += [("bad_magic", b"\0\0\0\0" + c2[4:]), ("trailing", c2 + b"\1\0\0\0")]
    aggs = [P.agg_expr("group_concat", 1, 1, None, P.slot_ref(0, 1, T.INT32))]
    out.append(("group_concat", P.Plan(P.agg(P.scan(0), 1, [], aggs), {0: [(1, T.INT32)], 1: [(1, int(T.STRING))]}).serialize()))
    aggs = [P.agg_expr("count_star", 1, 1)]
    out.append(("string_key", P.Plan(P.agg(P.scan(0), 1, [P.slot_ref(0, 1, T.STRING)], aggs),
                                     {0: [(1, int(T.STRING))], 1: [(1, int(T.INT64))]}).serialize()))
    return out


def _explain(L, desc):
    buf = ctypes.create_string_buffer(TEXT_LEN)
    rc = L.bkgpu_plan_explain(desc, len(desc), buf, TEXT_LEN)
    return rc, buf.value


def _run_threads(target, n):
    errors = []

    def wrap(i):
        try:
            target(i)
        except BaseException as e:  # noqa: BLE001 (reported by the main thread)
            errors.append(f"thread {i}: {e!r}")
    th = [threading.Thread(target=wrap, args=(i,), daemon=True) for i in range(n)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=300)
    assert not any(t.is_alive() for t in th), "a thread did not finish"
    assert not errors, errors[:5]


@pytest.fixture(scope="module")
def solo():
    """every descriptor's answer on one thread: (rc, text, bkgpu_last_error(NULL) after the call when it failed)"""
    L = _lib.lib()
    ref = {}
    for name, desc in _descriptors():
        rc, text = _explain(L, desc)
        ref[name] = (desc, rc, text, L.bkgpu_last_error(None) if rc else None)
    return ref


def test_the_descriptors_cover_success_and_several_failures(solo):
    ok = [n for n, (_, rc, _, _) in solo.items() if rc == _lib.OK]
    failed = {n: (rc, msg) for n, (_, rc, _, msg) in solo.items() if rc != _lib.OK}
    assert len(ok) >= 20 and len(failed) >= 8, (ok, failed)
    assert {rc for rc, _ in failed.values()} >= {_lib.EINVAL, _lib.EUNSUPPORTED}
    assert len({msg for _, msg in failed.values()}) >= 4, failed   # (distinct messages: a message from another thread would show)
    for n, (_, rc, text, msg) in solo.items():
        if rc != _lib.OK:
            assert text == msg and msg, (n, text, msg)   # explain writes the failure's message into `text` as well


def test_explain_from_eight_threads_equals_one_thread(solo):
    """8 threads lower the same mix of plans, each in its own shuffled order: every return code and text equals the single-threaded one"""
    L = _lib.lib()
    names = sorted(solo)
    barrier = threading.Barrier(THREADS)

    def worker(i):
        rng = random.Random(1000 + i)
        barrier.wait(timeout=60)
        for _ in range(ROUNDS):
            order = names[:]
            rng.shuffle(order)
            for n in order:
                desc, rc0, text0, _ = solo[n]
                rc, text = _explain(L, desc)
                assert (rc, text) == (rc0, text0), (n, rc, rc0, text[:200], text0[:200])
    _run_threads(worker, THREADS)


def test_last_error_is_the_calling_threads_own(solo):
    """bkgpu_last_error(NULL) after each call is the calling thread's last failure — a successful call leaves it as it was — and a new
    thread starts with an empty message, whatever the other threads failed with meanwhile"""
    L = _lib.lib()
    names = sorted(solo)
    barrier = threading.Barrier(THREADS)

    def worker(i):
        rng = random.Random(2000 + i)
        assert L.bkgpu_last_error(None) == b"", L.bkgpu_last_error(None)
        barrier.wait(timeout=60)
        mine = b""
        for _ in range(ROUNDS * len(names)):
            n = rng.choice(names)
            desc, rc0, _, msg0 = solo[n]
            rc, _ = _explain(L, desc)
            assert rc == rc0, (n, rc, rc0)
            if rc != _lib.OK:
                mine = msg0
            got = L.bkgpu_last_error(None)
            assert got == mine, (n, got, mine)
    _run_threads(worker, THREADS)
