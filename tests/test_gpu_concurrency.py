"""One device's workspace under concurrent callers (needs an H100: pytest -m gpu).

Every entry point on a device shares one set of cached buffers (the workspace, the Cheetah / Lion tables, the staging buffers, the
tables of the pipelined host encode). Calls are serialised on them by one event: each call waits for it on its own stream before its
first kernel and records it on that stream at its end. These tests drive that protocol from several streams and several host threads
and compare every output, size and canary with the oracle:

  a. an interleaved schedule of stream-ordered calls on 4 side streams and torch's default stream, enqueued first, synchronised once;
  b. every kind of synchronous entry point made while a stream-ordered call is still queued behind a sleep: it must wait for it;
  c. 8 host threads, each with its own stream and codec instance, mixing every kind of call;
  d. fresh allocations after density_b200_shutdown, host-buffer calls of growing size and then stream-ordered calls."""
import ctypes
import threading
import traceback

import numpy as np
import pytest

import oracle
import planted
from conftest import payload

pytestmark = pytest.mark.gpu

CANARY = 0xA5
CANARY_BYTES = 64
MIB = 1 << 20
ALG = {"chameleon": 0, "cheetah": 1, "lion": 2}
# torch.cuda._sleep spins for a number of SM clock cycles; DESIGN.md section 8 records 1980 MHz during timed steps, so 2e9 cycles is
# about one second at that clock and longer at a lower one. The sleeps that a check relies on (0.5 s and 2 s) only have to outlast a
# few enqueues, none of which waits for the device.
CYCLES_PER_S = 2_000_000_000
S300, S70K, S1M, S5M, S33M, S64M = 300, 70001, MIB + 7, 5 * MIB + 1021, 33 * MIB, 64 * MIB + 3


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device; there is no CPU fallback")
    return torch


@pytest.fixture(scope="module")
def lib(torch_cuda):
    import density_b200
    return density_b200.load()  # raises if the CUDA extension is missing


# ---- inputs and expected bytes ------------------------------------------------------------------------------------------------
_text = {}


def text(n, page=0):
    """n bytes of synthetic text starting at 64 KiB page `page` (generated on the device: the CPU generator is slow at 100+ MiB)."""
    if (n, page) not in _text:
        from density_b200 import synth
        _text[(n, page)] = synth.synth_text(n, device="cuda", first_page=page).cpu().numpy()
    return _text[(n, page)]


def make_input(kind, n, seed):
    """text, mixed and random inputs (text may and the other two do take copy mode), and prefixes of the planted corpora (cham5 and
    cham33 are quiet)"""
    if kind == "text":
        return text(n, seed)
    if kind in ("mixed", "random"):
        return payload(kind, n, seed)
    data = planted.corpus(kind)[0]
    assert n <= data.size
    return data[:n].copy()


def pipelined_input():
    """Host buffers of >= 96 MiB take the pipelined encode, in 64 MiB chunks: the planted corpus of 129 MiB + 7 B makes three, with
    plantings on both sides of each seam. It is quiet, so the encode stays on the pipeline instead of the whole-buffer fallback."""
    data = planted.corpus("cham129")[0]
    assert data.size >= 128 * MIB and quiet(data)
    return data


def quiet(data):
    """Chameleon encode path 1 has no fallback: it is only exact on inputs whose stream has no copy-mode block"""
    return oracle.encode("chameleon", data, return_copied=True)[1] == 0


def first_diff(a, b):
    k = min(a.size, b.size)
    d = np.flatnonzero(a[:k] != b[:k])
    return int(d[0]) if d.size else k


def check_bytes(what, n, got, want, tail):
    """the reported size, every byte of the output and a canary of CANARY_BYTES after the capacity"""
    assert n == want.size, f"{what}: size {n}, want {want.size}"
    assert (got[:n] == want).all(), f"{what}: first differing byte {first_diff(got[:n], want)}"
    assert tail.size >= CANARY_BYTES and (tail == CANARY).all(), f"{what}: wrote past the capacity"


def safe_size(alg, n):
    return oracle.safe_encode_buffer_size(alg, n)


def _sp(stream):
    return ctypes.c_void_p(stream.cuda_stream)


class DeviceCall:
    """One stream-ordered call with its device buffers: the output has CANARY_BYTES of canary after `cap`, and the size word starts
    at -1 so that a size that is never written shows up."""

    def __init__(self, torch, op, alg, path, n_in, cap, want):
        self.op, self.alg, self.path, self.n_in, self.cap, self.want = op, alg, path, n_in, cap, want
        self.d_in = torch.zeros(max(n_in, 1), dtype=torch.uint8, device="cuda")
        self.d_out = torch.full((cap + CANARY_BYTES,), CANARY, dtype=torch.uint8, device="cuda")
        self.d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")

    def reset(self):
        self.d_out.fill_(CANARY)
        self.d_sz.fill_(-1)

    def enqueue(self, lib, stream, d_in_ptr=None):
        f = lib.density_b200_encode_device_path if self.op == "enc" else lib.density_b200_decode_device_path
        rc = f(ALG[self.alg], self.d_in.data_ptr() if d_in_ptr is None else d_in_ptr, self.n_in, self.d_out.data_ptr(), self.cap,
               self.d_sz.data_ptr(), _sp(stream), self.path)
        assert rc == 0, f"{self.op} {self.alg} path {self.path}: rc {rc}, {lib.density_b200_last_error().decode()}"

    def check(self, what):
        out = self.d_out.cpu().numpy()
        check_bytes(what, int(self.d_sz.item()), out, self.want, out[self.cap:])


# ---- a. interleaved stream-ordered schedule ---------------------------------------------------------------------------------
# (op, alg, path, input kind, input bytes). "dec+" decodes the stream of the call before it, on that call's stream, from its d_out.
# The workspace grows three times in the middle (5 MiB, 33 MiB, 64 MiB + 3), and the calls after that are smaller again. "hold":
# a long sleep in front of this call, and the next call, on another stream, must still be queued behind it.
SCHEDULE = [
    ("enc", "chameleon", 0, "text", S300),
    ("enc", "cheetah", 1, "text", S70K),
    ("dec", "chameleon", 3, "mixed", S70K),
    ("enc", "lion", 3, "text", S300),
    ("dec", "cheetah", 0, "random", S1M),
    ("enc", "chameleon", 3, "random", S70K),
    ("dec", "lion", 0, "mixed", S70K),
    ("enc", "lion", 1, "cl1", S1M),
    ("enc", "chameleon", 0, "mixed", S5M),
    ("dec", "chameleon", 1, "text", S5M),
    ("enc", "cheetah", 0, "mixed", S5M),
    ("enc", "chameleon", 1, "cham33", S33M),
    ("enc", "cheetah", 3, "text", S300),
    ("dec", "cheetah", 1, "text", S33M),
    ("enc", "chameleon", 0, "text", S64M),
    ("dec+", "chameleon", 0, None, S64M),
    ("enc", "chameleon", 2, "mixed", S5M),
    ("dec", "chameleon", 1, "random", S1M, "hold"),
    ("enc", "chameleon", 0, "copy3", S1M),
    ("enc", "lion", 0, "text", S70K),
    ("dec+", "lion", 0, None, S70K),
    ("enc", "cheetah", 1, "random", S1M),
    ("dec+", "cheetah", 1, None, S1M),
    ("dec", "chameleon", 0, "copy3", S1M),
    ("enc", "chameleon", 1, "cham5", S1M),
    ("enc", "lion", 0, "mixed", S5M),
    ("enc", "cheetah", 0, "cl1", S1M),
    ("enc", "chameleon", 2, "text", S70K),
    ("dec", "chameleon", 3, "text", S300),
    ("enc", "chameleon", 0, "random", S300),
    ("dec", "cheetah", 0, "text", S70K),
    ("dec", "lion", 0, "text", S300),
]
SLEEPS = (0, 0, 0, CYCLES_PER_S // 2000, CYCLES_PER_S // 200, CYCLES_PER_S // 50)   # 0, 0.5, 5 and 20 ms
HOLD = CYCLES_PER_S // 2                                                             # 0.5 s


def test_schedule_covers_every_path():
    """The schedule's own promises: every listed path of every algorithm, at least 24 calls, the slow kernels (path 3, Lion decode)
    at 1 MiB or less, the 64 MiB call in the middle, smaller calls after it."""
    calls = {(op.rstrip("+"), alg, path) for op, alg, path, *_ in SCHEDULE}
    want = {("enc", "chameleon", p) for p in (0, 1, 2, 3)} | {("enc", a, p) for a in ("cheetah", "lion") for p in (0, 1, 3)} \
        | {("dec", "chameleon", p) for p in (0, 1, 3)} | {("dec", "cheetah", p) for p in (0, 1)} | {("dec", "lion", 0)}
    assert want <= calls, want - calls
    assert len(SCHEDULE) >= 24
    for op, alg, path, kind, n, *_ in SCHEDULE:
        if path == 3 or (op.startswith("dec") and alg == "lion"):
            assert n <= MIB, (op, alg, path, n)
    big = [k for k, e in enumerate(SCHEDULE) if e[4] == S64M]
    assert 0 < big[0] and big[-1] < len(SCHEDULE) - 8


def _plan_schedule(torch):
    """-> per call: (DeviceCall, pinned input or None, stream index, sleep cycles); 4 side streams + torch's default stream (index 4)"""
    rng = np.random.default_rng(20261017)
    calls = []
    for k, (op, alg, path, kind, n, *flags) in enumerate(SCHEDULE):
        if op == "dec+":
            enc_call, _, s, _ = calls[-1]
            want = oracle.decode(alg, enc_call.want, n)
            c = DeviceCall(torch, "dec", alg, path, enc_call.want.size, n, want)
            c.src, c.hold = enc_call, False    # reads enc_call.d_out
            calls.append((c, None, s, 0))
            continue
        data = make_input(kind, n, seed=k)
        if op == "enc":
            if alg == "chameleon" and path == 1:
                assert quiet(data), f"schedule call {k}: path 1 needs a quiet input"
            want = oracle.encode(alg, data)
            c = DeviceCall(torch, "enc", alg, path, n, safe_size(alg, n), want)
            host = data
        else:
            stream = oracle.encode(alg, data)
            assert (oracle.decode(alg, stream, n) == data).all()
            c = DeviceCall(torch, "dec", alg, path, stream.size, n, data)
            host = stream
        c.src, c.hold = None, bool(flags)
        s = int(rng.integers(0, 5))
        sleep = HOLD if c.hold else int(SLEEPS[int(rng.integers(0, len(SLEEPS)))])
        if calls and calls[-1][0].hold:
            sleep = 0                          # the call behind the held one: another stream, and nothing of its own to wait for
            if s == calls[-1][2]:
                s = (s + 1) % 5
        calls.append((c, torch.from_numpy(host).pin_memory(), s, sleep))
    return calls


def test_interleaved_stream_ordered_schedule(torch_cuda, lib):
    """Stream-ordered calls of every algorithm and path on 4 side streams and torch's default stream, enqueued with sleeps of
    different lengths in front of some of them so that the streams become ready in another order than the calls were enqueued. All
    are enqueued first and synchronised once; then every size, every byte and every canary is compared with the oracle."""
    torch = torch_cuda
    lib.density_b200_shutdown()                # nothing else is active: the schedule grows the workspace from nothing
    calls = _plan_schedule(torch)
    streams = [torch.cuda.Stream() for _ in range(4)] + [torch.cuda.default_stream()]
    torch.cuda.synchronize()                   # buffers filled, pinned inputs ready
    held = None
    for k, (c, host, s, sleep) in enumerate(calls):
        st = streams[s]
        with torch.cuda.stream(st):
            if sleep:
                torch.cuda._sleep(sleep)
            if c.src is None:
                c.d_in[:host.numel()].copy_(host, non_blocking=True)
                c.enqueue(lib, st)
            else:
                c.enqueue(lib, st, d_in_ptr=c.src.d_out.data_ptr())
        if held is not None:
            assert streams[held] is not st and not sleep
            assert not st.query(), f"call {k} finished before the call queued behind a {HOLD} cycle sleep on another stream"
            held = None
        if c.hold:
            held = s
    torch.cuda.synchronize()
    for k, (c, *_rest) in enumerate(calls):
        op, alg, path, kind, n, *_ = SCHEDULE[k]
        c.check(f"call {k}: {op} {alg} path {path} {kind} {n} B")


# ---- b. synchronous calls wait for stream-ordered work enqueued before them ---------------------------------------------------
SLEEP_B = 2 * CYCLES_PER_S                     # about 2 s


def _sync_cases(torch, lib):
    """-> [(name, call)]: each call makes one synchronous library call and returns a function that checks its result"""
    import density_b200
    from density_b200.codec import CodecInstance
    C = density_b200.CODECS
    cases = []

    def host_encode(alg, data, pinned):
        want = oracle.encode(alg, data)
        cap = safe_size(alg, data.size)
        pipelined = alg == "chameleon" and data.size >= 96 * MIB
        if pinned:
            pinned_bufs = (torch.from_numpy(data).pin_memory(), torch.empty(cap + CANARY_BYTES, dtype=torch.uint8).pin_memory())
            inp, out = (b.numpy() for b in pinned_bufs)
        else:
            inp, out = data, np.empty(cap + CANARY_BYTES, dtype=np.uint8)

        def call():
            out[:] = CANARY
            n = C[alg].encode(inp, out[:cap])
            # 1 right after a pipelined encode that stayed quiet, without touching the device (for other encodes it synchronises the
            # device, which would hide a call that did not wait)
            took_pipeline = pipelined and lib.density_b200_last_encode_was_fast() == 1

            def check(what):
                check_bytes(what, n, out, want, out[cap:])
                assert took_pipeline or not pipelined, f"{what}: the encode did not complete on the pipelined path"
            return check
        return call

    def host_decode(alg, data):
        stream = oracle.encode(alg, data)
        out = np.empty(data.size + CANARY_BYTES, dtype=np.uint8)

        def call():
            out[:] = CANARY
            n = C[alg].decode(stream, out[:data.size])
            return lambda what: check_bytes(what, n, out, data, out[data.size:])
        return call

    text_1m = text(S1M, 3)
    big = pipelined_input()
    cases.append(("chameleon_encode, 1 MiB host buffers", host_encode("chameleon", text_1m, False)))
    cases.append(("chameleon_encode, 129 MiB pinned host buffers (pipelined)", host_encode("chameleon", big, True)))
    cases.append(("chameleon_encode, 129 MiB pageable host buffers (pipelined)", host_encode("chameleon", big, False)))
    cases.append(("cheetah_decode, host buffers", host_decode("cheetah", make_input("mixed", S5M, 4))))
    cases.append(("lion_encode, host buffers", host_encode("lion", make_input("cl1", S1M, 0), False)))

    inst_data = make_input("copy3", S1M, 0)
    inst_stream = oracle.Codec("chameleon").encode(inst_data)
    enc_inst, dec_inst = CodecInstance("chameleon"), CodecInstance("chameleon")
    inst_out = np.empty(safe_size("chameleon", inst_data.size) + CANARY_BYTES, dtype=np.uint8)

    def inst_encode():
        enc_inst.clear_state()
        inst_out[:] = CANARY
        n = enc_inst.encode(inst_data, inst_out[:inst_out.size - CANARY_BYTES])
        return lambda what: check_bytes(what, n, inst_out, inst_stream, inst_out[-CANARY_BYTES:])

    def inst_decode():
        dec_inst.clear_state()
        out = np.full(inst_data.size + CANARY_BYTES, CANARY, dtype=np.uint8)
        n = dec_inst.decode(inst_stream, out[:inst_data.size])
        return lambda what: check_bytes(what, n, out, inst_data, out[inst_data.size:])
    cases.append(("CodecInstance.encode", inst_encode))
    cases.append(("CodecInstance.decode", inst_decode))

    dev_data = make_input("random", S5M, 8)
    dev_want = oracle.encode("cheetah", dev_data)
    d_in = torch.from_numpy(dev_data).cuda()
    d_out = torch.empty(safe_size("cheetah", dev_data.size) + CANARY_BYTES, dtype=torch.uint8, device="cuda")

    def dev_symbol():
        d_out.fill_(CANARY)
        n = lib.cheetah_encode(d_in.data_ptr(), dev_data.size, d_out.data_ptr(), d_out.numel() - CANARY_BYTES)

        def check(what):
            out = d_out.cpu().numpy()
            check_bytes(what, n, out, dev_want, out[-CANARY_BYTES:])
        return check
    cases.append(("cheetah_encode, device pointers", dev_symbol))
    return cases, (enc_inst, dec_inst)


def test_sync_calls_wait_for_stream_ordered_work(torch_cuda, lib):
    """A synchronous call may only start on the workspace when the stream-ordered call enqueued before it has released it. Side stream
    A holds a ~2 s sleep followed by an encode; the synchronous call is made while A's encode is still pending, and when it returns A
    must be done. The pipelined host encode (>= 96 MiB host buffers) is covered with pinned and with pageable buffers."""
    torch = torch_cuda
    cases, instances = _sync_cases(torch, lib)
    a_inputs = [("chameleon", text(S5M, 11)), ("cheetah", make_input("cl1", S1M, 0)), ("lion", make_input("mixed", S1M, 12))]
    a_calls = []
    for alg, data in a_inputs:
        c = DeviceCall(torch, "enc", alg, 0, data.size, safe_size(alg, data.size), oracle.encode(alg, data))
        c.d_in.copy_(torch.from_numpy(data))
        a_calls.append(c)
    big = DeviceCall(torch, "enc", "chameleon", 0, S64M, safe_size("chameleon", S64M), oracle.encode("chameleon", text(S64M, 7)))
    big.d_in.copy_(torch.from_numpy(text(S64M, 7)))
    A = torch.cuda.Stream()
    torch.cuda.synchronize()
    # warm-up: every buffer the calls below use reaches its size now (a buffer that grows frees the old one, and cudaFree waits for
    # the whole device, which would let a call that does not take the workspace pass)
    big.enqueue(lib, A)
    for c in a_calls:
        c.enqueue(lib, A)
    A.synchronize()
    for c in [big] + a_calls:
        c.check(f"warm-up: {c.alg} device encode of {c.n_in} B")
    for name, call in cases:
        call()(f"warm-up: {name}")
    for k, (name, call) in enumerate(cases):
        a = a_calls[k % len(a_calls)]
        a.reset()
        torch.cuda.synchronize()
        with torch.cuda.stream(A):
            torch.cuda._sleep(SLEEP_B)
        a.enqueue(lib, A)
        assert not A.query(), f"{name}: precondition: the encode on A should still be queued behind the sleep"
        check = call()
        assert A.query(), f"{name} returned while the stream-ordered encode enqueued before it was still pending"
        check(name)
        a.check(f"{name}: the {a.alg} encode on A")
    for inst in instances:
        inst.close()


# ---- c. host threads ----------------------------------------------------------------------------------------------------------
THREADS = 8
STEPS = 20


def _thread_plan(t):
    """seeded steps of thread t, with the oracle's bytes computed up front"""
    rng = np.random.default_rng(7000 + t)
    algs = ("chameleon", "cheetah", "lion")
    steps = []
    for k in range(STEPS):
        kind = ("dev", "host", "devptr", "inst")[int(rng.integers(0, 4))]
        alg = algs[int(rng.integers(0, 3))]
        src = ("text", "mixed", "random", "cl1" if alg != "chameleon" else "copy3")[int(rng.integers(0, 4))]
        sizes = (S300, 4099, S70K) if alg == "lion" and kind != "host" else (S300, 4099, S70K, S1M)
        n = int(sizes[int(rng.integers(0, len(sizes)))])
        seed = 100 * t + k
        if kind == "inst":
            alg = algs[t % 3]
            data = make_input(src, 3 * S70K, seed)
            cuts = sorted(int(x) for x in rng.integers(1, data.size, 2))
            pieces = [data[:cuts[0]], data[cuts[0]:cuts[1]], data[cuts[1]:]]
            ref = oracle.Codec(alg)
            steps.append(("inst", alg, pieces, [ref.encode(p) for p in pieces]))
            continue
        data = make_input(src, n, seed)
        steps.append((kind, alg, data, oracle.encode(alg, data), bool(rng.integers(0, 2))))
    if t == 0:      # calls that must fail: an encode into one byte less than the stream, a decode truncated inside a signature
        data = text(S70K, 21)
        want = oracle.encode("chameleon", data)
        assert oracle.decode("chameleon", want[:5], data.size).size == 0
        for k in (5, 12):
            steps.insert(k, ("fail_enc", "chameleon", data, want, False))
        steps.insert(17, ("fail_dec", "chameleon", data, want, False))
    return steps


def _run_thread(torch, lib, t, steps, errors):
    import density_b200
    from density_b200.codec import CodecInstance
    C = density_b200.CODECS
    try:
        s = torch.cuda.Stream()
        inst = CodecInstance(("chameleon", "cheetah", "lion")[t % 3])

        def ok(what):
            err = lib.density_b200_last_error()
            assert err == b"", f"thread {t}, {what}: last_error {err!r} after a successful call"

        for k, (kind, alg, *rest) in enumerate(steps):
            what = f"thread {t} step {k}: {kind} {alg}"
            if kind == "inst":
                pieces, wants = rest
                inst.clear_state()
                streams = []
                for j, (p, w) in enumerate(zip(pieces, wants)):
                    out = np.full(safe_size(alg, p.size) + CANARY_BYTES, CANARY, dtype=np.uint8)
                    n = inst.encode(p, out[:out.size - CANARY_BYTES])
                    ok(what)
                    check_bytes(f"{what} encode piece {j}", n, out, w, out[-CANARY_BYTES:])
                    streams.append(out[:n].copy())
                inst.clear_state()
                for j, (p, st) in enumerate(zip(pieces, streams)):
                    out = np.full(p.size + CANARY_BYTES, CANARY, dtype=np.uint8)
                    n = inst.decode(st, out[:p.size])
                    ok(what)
                    check_bytes(f"{what} decode piece {j}", n, out, p, out[p.size:])
                continue
            data, want, flip = rest
            cap = safe_size(alg, data.size)
            if kind == "dev":
                with torch.cuda.stream(s):
                    enc = DeviceCall(torch, "enc", alg, 0, data.size, cap, want)
                    dec = DeviceCall(torch, "dec", alg, 0, want.size, data.size, data)
                    enc.d_in.copy_(torch.from_numpy(data).pin_memory(), non_blocking=True)
                    enc.enqueue(lib, s)
                    ok(what)
                    dec.enqueue(lib, s, d_in_ptr=enc.d_out.data_ptr())
                    ok(what)
                s.synchronize()
                enc.check(f"{what} stream-ordered encode")
                dec.check(f"{what} stream-ordered decode")
            elif kind == "host":
                out = np.full(cap + CANARY_BYTES, CANARY, dtype=np.uint8)
                n = C[alg].encode(data, out[:cap])
                ok(what)
                check_bytes(f"{what} host encode", n, out, want, out[cap:])
                back = np.full(data.size + CANARY_BYTES, CANARY, dtype=np.uint8)
                m = C[alg].decode(want if flip else out[:n].copy(), back[:data.size])
                ok(what)
                check_bytes(f"{what} host decode", m, back, data, back[data.size:])
            elif kind == "devptr":
                with torch.cuda.stream(s):
                    d_in = torch.from_numpy(data).cuda()
                    d_out = torch.full((cap + CANARY_BYTES,), CANARY, dtype=torch.uint8, device="cuda")
                    d_enc = torch.from_numpy(want).cuda()
                    d_dec = torch.full((data.size + CANARY_BYTES,), CANARY, dtype=torch.uint8, device="cuda")
                n = getattr(lib, f"{alg}_encode")(d_in.data_ptr(), data.size, d_out.data_ptr(), cap)
                ok(what)
                m = getattr(lib, f"{alg}_decode")(d_enc.data_ptr(), want.size, d_dec.data_ptr(), data.size)
                ok(what)
                o = d_out.cpu().numpy()
                check_bytes(f"{what} device-pointer encode", n, o, want, o[cap:])
                o = d_dec.cpu().numpy()
                check_bytes(f"{what} device-pointer decode", m, o, data, o[data.size:])
                s.synchronize()
            elif kind == "fail_enc":
                out = np.full(want.size + CANARY_BYTES, CANARY, dtype=np.uint8)
                n = lib.chameleon_encode(data.ctypes.data, data.size, out.ctypes.data, want.size - 1)
                err = lib.density_b200_last_error()
                assert n == 0 and err != b"", f"{what}: an encode into one byte less than the stream returned {n}, last_error {err!r}"
                assert (out[want.size - 1:] == CANARY).all(), f"{what}: wrote past the capacity"
            elif kind == "fail_dec":
                out = np.full(data.size + CANARY_BYTES, CANARY, dtype=np.uint8)
                cut = want[:5].copy()
                m = lib.chameleon_decode(cut.ctypes.data, cut.size, out.ctypes.data, data.size)
                err = lib.density_b200_last_error()
                assert m == 0 and err != b"", f"{what}: a stream cut inside its first signature decoded to {m} bytes, last_error {err!r}"
        inst.close()
    except BaseException:
        errors.append(f"thread {t}:\n{traceback.format_exc()}")


def test_host_threads_share_the_workspace(torch_cuda, lib):
    """8 host threads, each with its own torch stream and codec instance, run seeded steps side by side (ctypes releases the GIL
    during a call): stream-ordered encode and decode waited for through the thread's stream only, the synchronous symbols with host
    and with device pointers, and three-piece instance continuations against oracle.Codec. Thread 0 also makes calls that must fail
    and checks that its thread-local last error is set; every successful call leaves it empty."""
    torch = torch_cuda
    plans = [_thread_plan(t) for t in range(THREADS)]
    errors = []
    threads = [threading.Thread(target=_run_thread, args=(torch, lib, t, plans[t], errors), daemon=True) for t in range(THREADS)]
    for th in threads:
        th.start()
    for th in threads:
        th.join(timeout=600)
    assert not any(th.is_alive() for th in threads), "a thread did not finish within 600 s (deadlock?)"
    torch.cuda.synchronize()
    assert not errors, "\n".join(errors)


# ---- d. fresh allocations ----------------------------------------------------------------------------------------------------
def test_fresh_allocations_after_shutdown(torch_cuda, lib):
    """After density_b200_shutdown every cached buffer is allocated afresh: host-buffer calls of growing size (the last one pipelined)
    allocate and grow the staging buffers, the workspace and the pipeline's tables, each zero-filled on the stream that uses it
    next; stream-ordered calls on side streams follow. Every result must equal the oracle's."""
    import density_b200
    torch = torch_cuda
    C = density_b200.CODECS
    torch.cuda.synchronize()
    lib.density_b200_shutdown()
    host_steps = [("enc", "cheetah", text(S300, 30)), ("dec", "chameleon", make_input("mixed", S70K, 31)),
                  ("enc", "lion", make_input("cl1", S1M, 0)), ("dec", "cheetah", make_input("random", S5M, 32)),
                  ("enc", "chameleon", make_input("copy3", S1M, 0)), ("enc", "chameleon", text(S33M, 33)),
                  ("enc", "chameleon", pipelined_input())]
    for op, alg, data in host_steps:
        what = f"host {op} {alg} {data.size} B"
        want = oracle.encode(alg, data)
        if op == "enc":
            cap = safe_size(alg, data.size)
            out = np.full(cap + CANARY_BYTES, CANARY, dtype=np.uint8)
            check_bytes(what, C[alg].encode(data, out[:cap]), out, want, out[cap:])
        else:
            out = np.full(data.size + CANARY_BYTES, CANARY, dtype=np.uint8)
            check_bytes(what, C[alg].decode(want, out[:data.size]), out, data, out[data.size:])
    assert lib.density_b200_last_encode_was_fast() == 1, "the 129 MiB host encode did not complete on the pipelined path"
    streams = [torch.cuda.Stream() for _ in range(2)]
    dev_steps = [("enc", "chameleon", 0, text(S64M, 34)), ("dec", "cheetah", 1, text(S33M, 35)),
                 ("enc", "lion", 0, make_input("mixed", S5M, 36)), ("dec", "chameleon", 0, make_input("copy3", S1M, 0))]
    calls = []
    for k, (op, alg, path, data) in enumerate(dev_steps):
        stream = oracle.encode(alg, data)
        if op == "enc":
            c = DeviceCall(torch, "enc", alg, path, data.size, safe_size(alg, data.size), stream)
            host = data
        else:
            c = DeviceCall(torch, "dec", alg, path, stream.size, data.size, data)
            host = stream
        calls.append((c, torch.from_numpy(host).pin_memory()))
    torch.cuda.synchronize()
    for k, (c, host) in enumerate(calls):
        st = streams[k % 2]
        with torch.cuda.stream(st):
            c.d_in[:host.numel()].copy_(host, non_blocking=True)
            c.enqueue(lib, st)
    torch.cuda.synchronize()
    for (op, alg, path, data), (c, _) in zip(dev_steps, calls):
        c.check(f"stream-ordered {op} {alg} path {path} {data.size} B")
