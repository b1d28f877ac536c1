"""Every sharded NCCL driver of libdensity_b200.so at W = 2..8 ranks on ONE H100 (pytest -m gpu), through the loopback collective
library (tests/loopback_nccl.cpp) installed with density_b200_test_set_nccl_library.

The single-GPU multi-rank tests run the phase functions with the exchanges and folds done in Python; this file runs the C++ drivers
themselves, so the in-driver folds (cham_rank_fold_k, cl_rank_fold_k, cl_prev_quad_k, chee_cmap_rank_fold), the seam verdict over
W rows, the per-rank exchange slots, the piece flags of the stream decoders and the grouped gather of the pieces all run at rank > 0.

W density_b200_sharded handles live in this process, each created and driven on its own thread (ctypes releases the GIL), and EVERY
rank passes the same CUDA stream: the persistent kernels of one rank never share the GPU with another rank's, the loopback only
enqueues device-to-device copies, and nothing on the device waits for the host, so a driver that issues its collectives in the wrong
order fails with a bounded host-side timeout instead of hanging the GPU. Every call checks that rc, *d_flags and *d_total_size agree
on all ranks, that the canaries behind every cap and gather_cap hold, and that each rank's collective sequence (the loopback's call
log) is the one include/density_b200.h states for the driver."""
import ctypes
import threading
import time

import numpy as np
import pytest

import loopback as lb
import oracle
from conftest import payload, splitmix_bytes

pytestmark = pytest.mark.gpu

MIB = 1 << 20
CANARY = 0xA5
OK, ECAPACITY, EARG = 0, 2, 4
ALG = {"chameleon": 0, "cheetah": 1, "lion": 2}


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device; there is no CPU fallback")
    import density_b200
    lib = density_b200.load()
    so, L = lb.build(tmp_path_factory.mktemp("loopback"))
    L.loopback_set_timeout_ms(20000)
    assert lib.density_b200_test_set_nccl_library(so.encode()) == OK, lib.density_b200_last_error()
    yield torch, lib, L
    assert lib.density_b200_test_set_nccl_library(None) == OK, lib.density_b200_last_error()


def _p(t):
    return t.data_ptr() if t is not None and t.numel() else None


class Ranks:
    """W handles on one communicator of the loopback; run() calls one driver on every rank at once, each on its own thread."""

    def __init__(self, env, world):
        self.torch, self.lib, self.L = env
        self.world = world
        uid = (ctypes.c_uint8 * 128)()
        assert self.lib.density_b200_sharded_unique_id(uid) == OK, self.lib.density_b200_last_error()
        self.h = [None] * world
        self._threads(lambda r: self.h.__setitem__(r, self.lib.density_b200_sharded_create(uid, r, world)))
        assert all(self.h), "density_b200_sharded_create failed"
        self.stream = ctypes.c_void_p(self.torch.cuda.current_stream().cuda_stream)

    def _threads(self, fn, ranks=None):
        ranks = range(self.world) if ranks is None else ranks
        out, errs = {}, []

        def work(r):
            try:
                out[r] = fn(r)
            except BaseException as e:      # noqa: BLE001 -- reported below
                errs.append((r, e))
        ts = [threading.Thread(target=work, args=(r,)) for r in ranks]
        for t in ts:
            t.start()
        for t in ts:
            t.join(120)
        assert not any(t.is_alive() for t in ts), "a rank did not return"
        assert not errs, errs
        return [out[r] for r in ranks]

    def run(self, call, ranks=None):
        """call(r, handle, stream) -> rc on every rank at once. Returns [(rc, last error)] per rank; waits for the stream."""
        self.L.loopback_log_clear()
        got = self._threads(lambda r: (call(r, self.h[r], self.stream), self.lib.density_b200_last_error().decode()), ranks)
        self.torch.cuda.synchronize()
        return got

    def logs(self, ranks=None):
        return [lb.call_log(self.L, r) for r in (range(self.world) if ranks is None else ranks)]

    def close(self):
        for h in self.h:
            if h:
                self.lib.density_b200_sharded_destroy(h)
        self.h = []

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def ag(*counts):
    return [(lb.ALLGATHER, c, lb.UINT32, -1) for c in counts]


def check_logs(R, want_ag, sizes=None, root=-1):
    """Every rank's call log = want_ag (the all-gathers), then its side of the gather of the pieces to `root`."""
    for r, log in enumerate(R.logs()):
        want = list(want_ag)
        if root >= 0 and r == root:
            want += [(lb.RECV, sizes[p], lb.UINT8, p) for p in range(R.world) if p != root and sizes[p]]
        elif root >= 0 and sizes[r]:
            want += [(lb.SEND, sizes[r], lb.UINT8, root)]
        assert log == want, (r, log[:8], want[:8], len(log), len(want))


def same(xs, what):
    assert all(x == xs[0] for x in xs), (what, xs)
    return xs[0]


# ---- the encoders ---------------------------------------------------------------------------------------------------------------------
def encode(env, alg, shards, driver="plain", gather_root=-1, gather_cap=None):
    """One sharded encode of `shards` (numpy, one per rank) through density_b200_encode_sharded[_cl|_protected] on fresh handles,
    with the per-call checks. Returns a dict: rc, err (per rank), elapsed, R_logs, and with rc 0 flags, total, pieces, gathered."""
    torch, lib, _ = env
    W = len(shards)
    safe = getattr(lib, f"{alg}_safe_encode_buffer_size")
    caps = [safe(s.size) for s in shards]
    d_in = [torch.from_numpy(s.copy()).cuda() if s.size else None for s in shards]
    d_out = [torch.full((c + 64,), CANARY, dtype=torch.uint8, device="cuda") for c in caps]
    d_sz = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    d_fl = [torch.full((1,), -1, dtype=torch.int32, device="cuda") for _ in range(W)]
    d_tot = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    gcap = sum(caps) if gather_cap is None else gather_cap
    d_g = torch.full((gcap + 64,), CANARY, dtype=torch.uint8, device="cuda") if gather_root >= 0 else None

    def call(r, h, st):
        g = (_p(d_g), gcap) if r == gather_root else (None, 0)
        common = (_p(d_in[r]), shards[r].size, _p(d_out[r]), caps[r], _p(d_sz[r]), _p(d_fl[r]), _p(d_tot[r]), gather_root, *g, st)
        if driver == "cl":
            return lib.density_b200_encode_sharded_cl(h, ALG[alg], *common)
        if driver == "protected":
            return lib.density_b200_encode_sharded_protected(h, *common)
        return lib.density_b200_encode_sharded(h, *common)

    with Ranks(env, W) as R:
        t0 = time.monotonic()
        res = R.run(call)
        elapsed = time.monotonic() - t0
        rc = same([x[0] for x in res], "rc")
        for r in range(W):
            assert bool((d_out[r][caps[r]:] == CANARY).all()), f"rank {r} wrote past cap"
        if d_g is not None:
            assert bool((d_g[gcap:] == CANARY).all()), "the gather wrote past gather_cap"
        out = {"rc": rc, "err": [x[1] for x in res], "elapsed": elapsed, "R_logs": R.logs()}
        if rc == OK:
            out["flags"] = same([int(f.item()) for f in d_fl], "flags")
            out["total"] = same([int(t.item()) for t in d_tot], "total")
            sizes = [int(s.item()) for s in d_sz]
            out["pieces"] = [d_out[r][:sizes[r]].cpu().numpy() for r in range(W)]
            if not out["flags"]:
                assert sum(sizes) == out["total"]
            out["gathered"] = d_g[:out["total"]].cpu().numpy() if d_g is not None else None
            if driver == "cl":
                wp = lib.density_b200_cl_table_words(ALG[alg], 0)
                wc = lib.density_b200_cl_table_words(ALG[alg], 1)
                want = ag(2, wp, wc, 8)
            elif driver == "protected":
                want = ag(2) + ag(65536, 200, 4) * lib.density_b200_prot_round_budget() + ag(8)
            else:
                want = ag(65536, 8)
            check_logs(R, want, sizes, gather_root)
    return out


def cut(data, cuts):
    return [data[cuts[r]:cuts[r + 1]] for r in range(len(cuts) - 1)]


def check_encode(env, alg, data, cuts, driver="plain", gather_root=-1, want=None):
    want = oracle.encode(alg, data) if want is None else want
    o = encode(env, alg, cut(data, cuts), driver, gather_root)
    assert o["rc"] == OK, o["err"]
    assert o["flags"] == 0, cuts
    cat = np.concatenate(o["pieces"])
    assert o["total"] == want.size and cat.size == want.size and (cat == want).all(), cuts
    if gather_root >= 0:
        assert (o["gathered"] == want).all()
    return o


def text(n, first_page=0):
    """Synthetic text. Chameleon's quiet-only paths take first_page 0, whose blocks never meet the protection automaton; other pages
    can start with two incompressible blocks, which those paths refuse."""
    from density_b200 import synth
    return synth.synth_text(n, first_page=first_page).numpy()


def ragged(data, world, seed):
    """(data cut short, cuts): unequal 256-byte multiples, an empty middle shard (world >= 4, and world 3 with an even seed) and a last
    shard of 1-3 bytes (otherwise)."""
    rng = np.random.default_rng(seed)
    tail = 1 + seed % 3
    body = (data.size - tail) // 256
    if world == 3 and seed % 2 == 0:
        c = 256 * int(rng.integers(1, body))
        return data, [0, c, c, data.size]
    inner = sorted(int(v) for v in rng.choice(np.arange(1, body), max(world - 3, 1) if world > 2 else 0, replace=False))
    if world > 3:
        inner.insert(len(inner) // 2 + 1, inner[len(inner) // 2])     # an empty shard after the middle one
    cuts = [0] + [256 * b for b in inner] + [256 * body, 256 * body + tail]
    return data[:cuts[-1]], cuts


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_encode_sharded_ragged_shards_and_every_gather_root(env, world):
    data = text(3 * MIB + 2 + 4099 * world)
    for k, root in enumerate(sorted({-1, 0, world // 2, world - 1})):
        d, cuts = ragged(data, world, k)
        check_encode(env, "chameleon", d, cuts, gather_root=root)


@pytest.mark.parametrize("world", [2, 4])
def test_encode_sharded_gather_at_exactly_the_stream_length(env, world):
    data, cuts = ragged(text(2 * MIB + 3 + 777 * world), world, 3)
    want = oracle.encode("chameleon", data)
    o = encode(env, "chameleon", cut(data, cuts), gather_root=world - 1, gather_cap=want.size)
    assert o["rc"] == OK and o["flags"] == 0 and (o["gathered"] == want).all()


def test_encode_sharded_noise_in_one_shard_is_refused_on_every_rank(env):
    data = text(2 * MIB, first_page=4)
    data[MIB:MIB + 64 * 1024] = splitmix_bytes(64 * 1024, 5)
    o = encode(env, "chameleon", cut(data, [0, MIB - 256 * 100, MIB + 256 * 500, data.size]))
    assert o["rc"] == OK and o["flags"] != 0


def test_encode_sharded_gather_capacity_short_fails_on_every_rank(env):
    """gather_cap one byte below the stream length: every rank returns ECAPACITY within a second (none posts a send the root never
    receives), and nothing is written past gather_cap."""
    data, cuts = ragged(text(2 * MIB + 5), 3, 1)
    for driver, alg in (("plain", "chameleon"), ("protected", "chameleon"), ("cl", "cheetah")):
        w = check_encode(env, alg, data, cuts, driver, gather_root=2)["gathered"]      # also loads the kernels
        for root in (0, 2):
            o = encode(env, alg, cut(data, cuts), driver, gather_root=root, gather_cap=w.size - 1)
            assert o["rc"] == ECAPACITY, (driver, root, o["err"])
            assert o["elapsed"] < 1.0, o["elapsed"]
            assert all("gather buffer too small" in e for e in o["err"]), o["err"]
            assert not any(e[0] in (lb.SEND, lb.RECV) for log in o["R_logs"] for e in log)


def test_encode_sharded_null_gather_on_the_root_before_any_collective(env):
    torch, lib, L = env
    d_in = torch.from_numpy(text(MIB)).cuda()
    cap = lib.chameleon_safe_encode_buffer_size(MIB)
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    s = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(3)]
    with Ranks(env, 2) as R:
        for fn in ("density_b200_encode_sharded", "density_b200_encode_sharded_protected"):
            res = R.run(lambda r, h, st: getattr(lib, fn)(h, d_in.data_ptr(), MIB, d_out.data_ptr(), cap, s[0].data_ptr(), s[1].data_ptr(),
                                                          s[2].data_ptr(), 1, None, 0, st), ranks=[1])
            assert res[0][0] == EARG and "d_gather" in res[0][1]
            assert R.logs([1]) == [[]]
        res = R.run(lambda r, h, st: lib.density_b200_encode_sharded_cl(h, 1, d_in.data_ptr(), MIB, d_out.data_ptr(), cap, s[0].data_ptr(),
                                                                         s[1].data_ptr(), s[2].data_ptr(), 1, None, 0, st), ranks=[1])
        assert res[0][0] == EARG and R.logs([1]) == [[]]


@pytest.mark.parametrize("alg", ["cheetah", "lion"])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_encode_sharded_cl(env, alg, world):
    """Ragged shards with an empty one in front of the last: the last shard's previous quad comes from the nearest earlier shard that
    has one, not from the shard before it, and at world 4 not from the first shard either."""
    data = text(2 * MIB + 3, first_page=7)
    want = oracle.encode(alg, data)
    n = data.size
    cuts = {2: [0, 256 * 3001, n], 3: [0, 256 * 3001, 256 * 3001, n], 4: [0, 256 * 2000, 256 * 5001, 256 * 5001, n]}[world]
    check_encode(env, alg, data, cuts, "cl", gather_root=world - 1, want=want)
    d, cuts = ragged(data, world, world)
    check_encode(env, alg, d, cuts, "cl", gather_root=0)


@pytest.mark.parametrize("alg", ["cheetah", "lion"])
def test_encode_sharded_cl_copy_mode_after_rank0_is_refused(env, alg):
    t = text(2 * MIB, first_page=5)
    d = np.concatenate([t[:MIB], splitmix_bytes(MIB, 12)])
    for cuts in ([0, MIB, d.size], [0, MIB // 2, MIB, d.size]):
        o = encode(env, alg, cut(d, cuts), "cl")
        assert o["rc"] == OK and o["flags"] != 0


def _protected_corpora():
    """The inputs of test_gpu_sharded_protected_encode.py: noise, mixed data, text with noise bursts at the cuts, automaton states on
    the cuts, the copy decisions that feed each other across shards."""
    import protection as P
    from density_b200 import synth
    import test_gpu_sharded_protected_encode as T
    out = [(payload("random", 3 * MIB + 77, 1), T.cuts_at(3 * MIB + 77, 1111, 5003, 9999)),
           (synth.synth_mixed(4 * MIB).numpy(), T.cuts_at(4 * MIB, 8192))]
    data = T.text(2 * MIB)
    rnd = payload("random", 64 * 1024, 7)
    for i, b in enumerate([1000, 2501, 4097]):
        lo = [b * 256 - 2048, b * 256 - 1024, b * 256][i]
        data[lo:lo + 2048] = rnd[i * 8192:i * 8192 + 2048]
    out.append((data, T.cuts_at(data.size, 1000, 2501, 4097)))
    states = sorted(P.reachable_states())[:3]
    bld = P.Builder("chameleon", 33)
    cuts = [0]
    for st in states:
        bld.add("Z" * 40)
        b = next(b for b in range(bld.n + 1, bld.n + 2000) if b % 16 == st[3] and len(P.word_to(st[:3], b)) <= b - bld.n)
        bld.place(b, st[:3], "cut")
        cuts.append(b)
        bld.recover()
    bld.add("Z" * 20)
    d, _ = bld.realize()
    out.append((d, [c * 256 for c in cuts] + [d.size]))
    fb = T._feedback_input()
    out.append((fb, T.cuts_at(fb.size, 300, 620, 900)))
    return out


@pytest.mark.parametrize("world", [2, 3, 4])
def test_encode_sharded_protected(env, world):
    for data, cuts in _protected_corpora():
        inner = cuts[1:-1]
        if len(inner) >= world - 1:                   # the corpus' own cuts, thinned out to `world` shards
            inner = [inner[i * len(inner) // (world - 1)] for i in range(world - 1)]
        else:
            inner = inner + [data.size // 256 * (i + 1) // world * 256 for i in range(world - 1 - len(inner))]
        check_encode(env, "chameleon", data, [0] + sorted(inner) + [data.size], "protected", gather_root=world // 2)


def test_encode_sharded_protected_budget_too_small_is_refused(env):
    import test_gpu_sharded_protected_encode as T
    _, lib, _ = env
    data = T._feedback_input()
    cuts = T.cuts_at(data.size, 300, 620, 900)
    lib.density_b200_test_set_prot_rounds(1)
    try:
        o = encode(env, "chameleon", cut(data, cuts), "protected", gather_root=1)
        assert o["rc"] == OK and o["flags"] != 0 and o["total"] == 0
    finally:
        lib.density_b200_test_set_prot_rounds(0)


# ---- the decoders ---------------------------------------------------------------------------------------------------------------------
def decode(env, pieces, caps, alg="chameleon"):
    """density_b200_decode_sharded[_cheetah] of `pieces` on fresh handles, with the per-call checks. Returns (rc, flags, total, outs)."""
    torch, lib, _ = env
    W = len(pieces)
    d_in = [torch.from_numpy(np.ascontiguousarray(p)).cuda() if p.size else None for p in pieces]
    d_out = [torch.full((c + 64,), CANARY, dtype=torch.uint8, device="cuda") for c in caps]
    d_sz = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    d_fl = [torch.full((1,), -1, dtype=torch.int32, device="cuda") for _ in range(W)]
    d_tot = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    fn = lib.density_b200_decode_sharded if alg == "chameleon" else lib.density_b200_decode_sharded_cheetah
    with Ranks(env, W) as R:
        res = R.run(lambda r, h, st: fn(h, _p(d_in[r]), pieces[r].size, _p(d_out[r]), caps[r], _p(d_sz[r]), _p(d_fl[r]), _p(d_tot[r]), st))
        rc = same([x[0] for x in res], "rc")
        assert rc == OK, res
        for r in range(W):
            assert bool((d_out[r][caps[r]:] == CANARY).all()), f"rank {r} wrote past cap"
        flags = same([int(f.item()) for f in d_fl], "flags")
        total = same([int(t.item()) for t in d_tot], "total")
        if alg == "chameleon":
            want = ag(65536, 8)
        else:
            want = ag(lib.density_b200_cheetah_cmap_words()) + ag(131072, 4) * lib.density_b200_cheetah_decode_round_budget() + ag(8)
        check_logs(R, want)
        outs = [d_out[r][:max(int(d_sz[r].item()), 0)].cpu().numpy() for r in range(W)]
    return flags, total, outs


def check_decode_pieces(env, alg, data, cuts):
    """encode_sharded[_cl] of data cut at `cuts`, then decode_sharded[_cheetah] of the pieces: every rank gets its shard back."""
    shards = cut(data, cuts)
    o = encode(env, alg, shards, "plain" if alg == "chameleon" else "cl")
    assert o["rc"] == OK and o["flags"] == 0
    flags, total, outs = decode(env, o["pieces"], [max(s.size, 4) for s in shards], alg)
    assert flags == 0 and total == data.size
    for r, s in enumerate(shards):
        assert outs[r].size == s.size and (outs[r] == s).all(), r
    return o["pieces"]


@pytest.mark.parametrize("alg", ["chameleon", "cheetah"])
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_decode_sharded_pieces_of_the_encoders(env, alg, world):
    for seed in (world, world + 1):
        data = text(2 * MIB + 5 + 1237 * world, first_page=0 if alg == "chameleon" else 3 + world)
        check_decode_pieces(env, alg, *ragged(data, world, seed))


def test_decode_sharded_cheetah_rounds_budget_too_small_is_refused(env):
    _, lib, _ = env
    data = text(3 * MIB + 1001)
    cuts = [0, MIB, 2 * MIB, data.size]
    shards = cut(data, cuts)
    pieces = encode(env, "cheetah", shards, "cl")["pieces"]
    lib.density_b200_test_set_decode_rounds(1)
    try:
        flags, _, _ = decode(env, pieces, [s.size for s in shards], "cheetah")
        assert flags != 0
    finally:
        lib.density_b200_test_set_decode_rounds(40)


def test_decode_sharded_chameleon_copy_mode_piece_is_refused(env):
    """The pieces of a protected encode with copy-mode blocks in piece 1: the quiet-only decoder refuses them on every rank."""
    d = text(2 * MIB, first_page=6)
    d[MIB + 4096:MIB + 4096 + 64 * 1024] = splitmix_bytes(64 * 1024, 8)
    shards = cut(d, [0, MIB, d.size])
    o = encode(env, "chameleon", shards, "protected")
    assert o["rc"] == OK and o["flags"] == 0
    flags, _, _ = decode(env, o["pieces"], [s.size for s in shards])
    assert flags != 0


# ---- the stream decoders ------------------------------------------------------------------------------------------------------------
def decode_stream(env, stream, lay, alg):
    """density_b200_decode_sharded[_cheetah]_stream of `stream` in layout `lay` [(offset, n_range, n_halo)] on fresh handles. Returns
    (flags, total, outputs placed at their *d_out_offset, or None when refused)."""
    torch, lib, _ = env
    W = len(lay)
    mul = 2 if alg == "chameleon" else 16
    caps = [max(mul * (n + h), 4) for _, n, h in lay]
    bufs = [np.ascontiguousarray(stream[o:o + n + h]) for o, n, h in lay]
    d_in = [torch.from_numpy(b).cuda() if b.size else None for b in bufs]
    d_out = [torch.full((c + 64,), CANARY, dtype=torch.uint8, device="cuda") for c in caps]
    d_sz, d_off, d_tot = ([torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)] for _ in range(3))
    d_fl = [torch.full((1,), -1, dtype=torch.int32, device="cuda") for _ in range(W)]

    def call(r, h, st):
        o, n, hl = lay[r]
        tail = (_p(d_out[r]), caps[r], _p(d_sz[r]), _p(d_off[r]), _p(d_fl[r]), _p(d_tot[r]), st)
        if alg == "chameleon":
            return lib.density_b200_decode_sharded_stream(h, _p(d_in[r]), n, hl, *tail)
        return lib.density_b200_decode_sharded_cheetah_stream(h, _p(d_in[r]), n, hl, o, *tail)

    with Ranks(env, W) as R:
        res = R.run(call)
        rc = same([x[0] for x in res], "rc")
        assert rc == OK, res
        for r in range(W):
            assert bool((d_out[r][caps[r]:] == CANARY).all()), f"rank {r} wrote past cap"
        flags = same([int(f.item()) for f in d_fl], "flags")
        total = same([int(t.item()) for t in d_tot], "total")
        if alg == "chameleon":
            want = ag(2 * 266, 65536, 8)
        else:
            want = ag(2 * 142, lib.density_b200_cheetah_cmap_words()) + ag(131072, 4) * lib.density_b200_cheetah_decode_round_budget() + ag(8)
        check_logs(R, want)
        if flags:
            return flags, total, None
        out = np.full(total, 0x5A, np.uint8)
        for r in range(W):
            sz, off = int(d_sz[r].item()), int(d_off[r].item())
            assert 0 <= off and off + sz <= total
            out[off:off + sz] = d_out[r][:sz].cpu().numpy()
        offs = sorted((int(d_off[r].item()), int(d_sz[r].item())) for r in range(W))
        assert sum(s for _, s in offs) == total and all(a[0] + a[1] <= b[0] for a, b in zip(offs, offs[1:]))
    return flags, total, out


def check_stream(env, stream, data, lay, alg):
    flags, total, out = decode_stream(env, stream, lay, alg)
    assert flags == 0 and total == data.size, lay
    assert (out == data).all(), lay


def hand_layouts(total):
    """stream_ranges at W = 2, 3, 5, 8 and hand layouts with zero-length ranges: in the middle, and in front of the stream start."""
    from density_b200 import sharded
    from locate_model import CH, layout
    out = [sharded.stream_ranges(total, w) for w in (2, 3, 5, 8)]
    k = total // CH
    a = k // 3 * CH
    out.append(layout(total, [a, 0, 0, a, 0, total - 2 * a]))
    out.append(layout(total, [0, a, total - a]))                  # the stream start on rank 1
    out.append(layout(total, [0, 0, a, 0, total - a]))            # ... behind two empty ranges
    return out


@pytest.mark.parametrize("alg", ["chameleon", "cheetah"])
def test_decode_sharded_stream_layouts(env, alg):
    data = text(3 * MIB + 403, first_page=0 if alg == "chameleon" else 3)
    stream = oracle.encode(alg, data)
    for lay in hand_layouts(stream.size):
        check_stream(env, stream, data, lay, alg)


@pytest.mark.parametrize("alg", ["chameleon", "cheetah"])
def test_decode_sharded_stream_of_a_tiny_stream_over_eight_ranks(env, alg):
    from density_b200 import sharded
    data = text(3000, first_page=0 if alg == "chameleon" else 1)
    stream = oracle.encode(alg, data)
    check_stream(env, stream, data, sharded.stream_ranges(stream.size, 8), alg)


def test_decode_sharded_stream_copy_mode_is_refused_on_every_rank(env):
    from density_b200 import sharded
    t = text(2 * MIB, first_page=5)
    d = np.concatenate([t[:MIB], splitmix_bytes(256 * 1024, 12), t[MIB:]])
    for alg in ("chameleon", "cheetah"):
        stream = oracle.encode(alg, d)
        for w in (2, 3):
            flags, _, _ = decode_stream(env, stream, sharded.stream_ranges(stream.size, w), alg)
            assert flags != 0, (alg, w)
