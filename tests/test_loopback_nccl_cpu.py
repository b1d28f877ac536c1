"""The loopback collective library (tests/loopback_nccl.cpp) on host memory, one Python thread per rank (ctypes releases the GIL):
all-gather in place and out of place, grouped send / recv, and the bounded failures -- a count mismatch, a rank that never arrives,
a send nobody receives -- that the multi-rank GPU tests rely on to turn a driver's collective-order bug into an error instead of a
hang. These are the only tests that desynchronise the ranks on purpose, and they do it with host memory only."""
import ctypes
import threading
import time

import numpy as np
import pytest

import loopback as lb


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    _, L = lb.build(tmp_path_factory.mktemp("loopback"))
    L.loopback_set_host_copy(1)
    return L


@pytest.fixture(autouse=True)
def fresh(L):
    L.loopback_log_clear()
    yield
    L.loopback_set_timeout_ms(60000)


def run_ranks(L, world, body, join_s=30):
    """body(rank, comm) on `world` threads that share one fresh id; returns [result per rank]. Every comm is destroyed afterwards."""
    uid = lb.UniqueId()
    assert L.ncclGetUniqueId(ctypes.byref(uid)) == lb.OK
    out, errs = [None] * world, []

    def worker(r):
        comm = ctypes.c_void_p()
        try:
            rc = L.ncclCommInitRank(ctypes.byref(comm), world, uid, r)
            assert rc == lb.OK, L.ncclGetErrorString(rc)
            out[r] = body(r, comm)
        except BaseException as e:      # noqa: BLE001 -- reported on the main thread
            errs.append((r, e))
        finally:
            L.ncclCommDestroy(comm)

    ts = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(join_s)
    assert not any(t.is_alive() for t in ts), "a rank is still waiting"
    assert not errs, errs
    return out


def ptr(a, off=0):
    return ctypes.c_void_p(a.ctypes.data + int(off))


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("in_place", [False, True])
def test_all_gather(L, world, in_place):
    rng = np.random.default_rng(world)
    sends = [rng.integers(0, 2 ** 32, 37, dtype=np.uint32) for _ in range(world)]
    recvs = [np.zeros(37 * world, np.uint32) for _ in range(world)]

    def body(r, comm):
        out = []
        for k in range(3):                              # consecutive calls reuse the comm's rendezvous
            s = sends[r] + np.uint32(k)
            if in_place:
                recvs[r][37 * r:37 * (r + 1)] = s
                src = ptr(recvs[r], 4 * 37 * r)
            else:
                src = ptr(s)
            assert L.ncclAllGather(src, ptr(recvs[r]), 37, lb.UINT32, comm, None) == lb.OK
            out.append(recvs[r].copy())
        return out

    got = run_ranks(L, world, body)
    for k in range(3):
        want = np.concatenate([s + np.uint32(k) for s in sends])
        for r in range(world):
            assert (got[r][k] == want).all(), (r, k)
    for r in range(world):
        assert lb.call_log(L, r) == [(lb.ALLGATHER, 37, lb.UINT32, -1)] * 3


@pytest.mark.parametrize("world,root,sizes", [(2, 0, [5, 3]), (3, 1, [4, 0, 9]), (4, 3, [0, 7, 0, 1]), (5, 2, [11, 0, 6, 2000, 0]),
                                              (3, 0, [0, 0, 0])])
def test_grouped_gather_to_a_root(L, world, root, sizes):
    """The pattern of the sharded encoders' gather: every non-empty piece but the root's is sent to the root, which receives them at
    their prefix-sum offsets in one group; empty pieces post nothing."""
    rng = np.random.default_rng(sum(sizes))
    pieces = [rng.integers(0, 256, s, dtype=np.uint8) for s in sizes]
    offs = [0] + [int(v) for v in np.cumsum(sizes)]
    dest = np.full(offs[-1] + 16, 0xEE, np.uint8)

    def body(r, comm):
        assert L.ncclGroupStart() == lb.OK
        if r == root:
            dest[offs[r]:offs[r + 1]] = pieces[r]
            for p in range(world):
                if p != r and sizes[p]:
                    assert L.ncclRecv(ptr(dest, offs[p]), sizes[p], lb.UINT8, p, comm, None) == lb.OK
        elif sizes[r]:
            assert L.ncclSend(ptr(pieces[r]), sizes[r], lb.UINT8, root, comm, None) == lb.OK
        rc = L.ncclGroupEnd()
        assert rc == lb.OK, L.ncclGetErrorString(rc)

    run_ranks(L, world, body)
    assert (dest[:offs[-1]] == np.concatenate(pieces)).all() and (dest[offs[-1]:] == 0xEE).all()
    for r in range(world):
        if r == root:
            want = [(lb.RECV, sizes[p], lb.UINT8, p) for p in range(world) if p != r and sizes[p]]
        else:
            want = [(lb.SEND, sizes[r], lb.UINT8, root)] if sizes[r] else []
        assert lb.call_log(L, r) == want


def test_sends_between_one_pair_match_in_fifo_order(L):
    a, b = np.arange(10, dtype=np.uint8), np.arange(100, 120, dtype=np.uint8)
    ra, rb = np.zeros(10, np.uint8), np.zeros(20, np.uint8)

    def body(r, comm):
        assert L.ncclGroupStart() == lb.OK
        if r == 0:
            L.ncclSend(ptr(a), 10, lb.UINT8, 1, comm, None)
            L.ncclSend(ptr(b), 20, lb.UINT8, 1, comm, None)
        else:
            L.ncclRecv(ptr(ra), 10, lb.UINT8, 0, comm, None)
            L.ncclRecv(ptr(rb), 20, lb.UINT8, 0, comm, None)
        assert L.ncclGroupEnd() == lb.OK

    run_ranks(L, 2, body)
    assert (ra == a).all() and (rb == b).all()


def test_count_mismatch_fails_every_rank_at_once(L):
    """One rank all-gathers a different count: every rank gets ncclInvalidUsage long before the timeout, with a message that names the
    operation, the counts and the ranks that had arrived; the comm stays poisoned."""
    L.loopback_set_timeout_ms(20000)
    world = 3
    bufs = [np.zeros(8 * world, np.uint32) for _ in range(world)]

    def body(r, comm):
        t0 = time.monotonic()
        rc = L.ncclAllGather(ptr(bufs[r], 32 * r), ptr(bufs[r]), 9 if r == 2 else 8, lb.UINT32, comm, None)
        msg = L.ncclGetErrorString(rc).decode()
        rc2 = L.ncclAllGather(ptr(bufs[r], 32 * r), ptr(bufs[r]), 8, lb.UINT32, comm, None)
        return rc, msg, time.monotonic() - t0, rc2

    got = run_ranks(L, world, body)
    for rc, msg, dt, rc2 in got:
        assert rc == lb.INVALID_USAGE and rc2 == lb.INVALID_USAGE
        assert dt < 5, dt
        assert "ncclAllGather mismatch" in msg and "count 9" in msg and "count 8" in msg, msg


def test_a_rank_that_never_arrives_times_out(L):
    L.loopback_set_timeout_ms(500)
    world = 3
    bufs = [np.zeros(4 * world, np.uint32) for _ in range(world)]

    def body(r, comm):
        if r == 2:
            return None
        t0 = time.monotonic()
        rc = L.ncclAllGather(ptr(bufs[r], 16 * r), ptr(bufs[r]), 4, lb.UINT32, comm, None)
        return rc, L.ncclGetErrorString(rc).decode(), time.monotonic() - t0

    got = run_ranks(L, world, body)
    for rc, msg, dt in got[:2]:
        assert rc == lb.INTERNAL and 0.4 < dt < 5, (rc, dt)
        assert "timed out" in msg and "arrived:" in msg, msg
    assert any("arrived: 0 (count 4" in m and "1 (count 4" in m for _, m, _ in got[:2])


def test_a_send_nobody_receives_times_out(L):
    """What a gather root that returns early leaves behind: the senders' GroupEnd fails within the timeout with "unmatched send"."""
    L.loopback_set_timeout_ms(500)
    piece = np.arange(64, dtype=np.uint8)

    def body(r, comm):
        if r == 0:
            return None                                 # the root posts nothing
        t0 = time.monotonic()
        assert L.ncclGroupStart() == lb.OK
        assert L.ncclSend(ptr(piece), 64, lb.UINT8, 0, comm, None) == lb.OK
        rc = L.ncclGroupEnd()
        return rc, L.ncclGetErrorString(rc).decode(), time.monotonic() - t0

    got = run_ranks(L, 3, body)
    for rc, msg, dt in got[1:]:
        assert rc in (lb.INTERNAL, lb.INVALID_USAGE) and dt < 5, (rc, dt)
    assert any("unmatched send" in m for _, m, _ in got[1:]), got


def test_call_log_records_and_clears(L):
    bufs = [np.zeros(2 * 2 + 8, np.uint32) for _ in range(2)]

    def body(r, comm):
        L.ncclAllGather(ptr(bufs[r], 8 * r), ptr(bufs[r]), 2, lb.UINT32, comm, None)
        L.ncclGroupStart()
        if r == 0:
            L.ncclRecv(ptr(bufs[0], 16), 3, lb.UINT8, 1, comm, None)
        else:
            L.ncclSend(ptr(bufs[1], 16), 3, lb.UINT8, 0, comm, None)
        assert L.ncclGroupEnd() == lb.OK

    run_ranks(L, 2, body)
    assert lb.call_log(L, 0) == [(lb.ALLGATHER, 2, lb.UINT32, -1), (lb.RECV, 3, lb.UINT8, 1)]
    assert lb.call_log(L, 1) == [(lb.ALLGATHER, 2, lb.UINT32, -1), (lb.SEND, 3, lb.UINT8, 0)]
    L.loopback_log_clear()
    assert lb.call_log(L, 0) == [] and lb.call_log(L, 1) == []
