"""The phase order and the argument rule of the sharded encode shards and drivers (include/density_b200.h, "Sharded encode"; needs an
H100: pytest -m gpu).

The order matrix drives a Chameleon and a Cheetah / Lion shard to every stage it can reach and calls every entry there: an entry the
order forbids returns DENSITY_B200_EARG and enqueues nothing, one it allows succeeds. The argument checks give every entry and driver
each of its pointers misaligned (and NULL where NULL is not allowed): DENSITY_B200_EARG with nothing enqueued; the same shard or
world-1 driver then encodes with aligned pointers to the bytes the oracle writes."""
import ctypes

import numpy as np
import pytest

import oracle

pytestmark = pytest.mark.gpu

EARG = 4
ALG_ID = {"chameleon": 0, "cheetah": 1, "lion": 2}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device; there is no CPU fallback")
    return torch


@pytest.fixture(scope="module")
def lib(torch_cuda):
    import density_b200
    return density_b200.load()


@pytest.fixture
def budget(lib):
    """the round budget of the copy-map iteration, restored after the test"""
    yield lib.density_b200_test_set_prot_rounds
    lib.density_b200_test_set_prot_rounds(0)


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def text(n):
    from density_b200 import synth
    return synth.synth_text(n).numpy()


def with_noise(n):
    """text with a run of noise in the middle: the copy-map iteration has blocks to settle"""
    d = text(n)
    d[n // 3:n // 3 + 4096] = np.random.default_rng(7).integers(0, 256, 4096, dtype=np.uint8)
    return d


class Bufs:
    """one shard's device buffers: the input, the output, a table, a carry, words, transfers, the sizes, the seam words and the flags"""

    def __init__(self, torch, alg, data):
        self.data, self.alg = data, alg
        self.n = data.size
        self.cap = self.n + self.n // 8 + 4096           # above the safe encode size of every algorithm
        self.d_in = torch.from_numpy(data.copy()).cuda()
        self.d_out = torch.zeros(self.cap + 64, dtype=torch.uint8, device="cuda")
        self.table = torch.zeros(12 * 65536 + 2, dtype=torch.int32, device="cuda")
        self.carry = torch.zeros(12 * 65536 + 2, dtype=torch.int32, device="cuda")
        self.words = torch.zeros(64, dtype=torch.int32, device="cuda")
        self.transfers = torch.zeros(4096, dtype=torch.int32, device="cuda")
        self.size = torch.zeros(2, dtype=torch.int64, device="cuda")
        self.total = torch.zeros(2, dtype=torch.int64, device="cuda")
        self.seam = torch.zeros(10, dtype=torch.int32, device="cuda")
        self.flags = torch.zeros(2, dtype=torch.int32, device="cuda")
        self.i, self.o, self.t, self.c = self.d_in.data_ptr(), self.d_out.data_ptr(), self.table.data_ptr(), self.carry.data_ptr()
        self.w, self.tr, self.sz, self.sm = self.words.data_ptr(), self.transfers.data_ptr(), self.size.data_ptr(), self.seam.data_ptr()
        self.fl, self.tot = self.flags.data_ptr(), self.total.data_ptr()

    def encoded(self, torch):
        torch.cuda.synchronize()
        n = int(self.size[0].item())
        want = oracle.encode(self.alg, self.data)
        return n == want.size and bool((self.d_out[:n].cpu().numpy() == want).all())


def refused(lib, *calls):
    """every call returns DENSITY_B200_EARG and none of them enqueues a kernel"""
    before = lib.density_b200_kernel_launches()
    rcs = [c() for c in calls]
    assert rcs == [EARG] * len(calls)
    assert lib.density_b200_kernel_launches() == before


# ---- the Chameleon shard ------------------------------------------------------------------------------------------------------------
def cham_entries(lib, h, b, st):
    status = (ctypes.c_uint32 * 20)()
    return {
        "phase1": lambda: lib.density_b200_shard_phase1(h, b.i, b.n, 1, b.t, st),
        "phase2": lambda: lib.density_b200_shard_phase2(h, None, b.o, b.cap, b.sz, b.fl, st),
        "prot_phase1": lambda: lib.density_b200_shard_prot_phase1(h, b.i, b.n, 0, 1, b.t, st),
        "transfer": lambda: lib.density_b200_shard_prot_transfer(h, None, b.tr, st),
        "settle": lambda: lib.density_b200_shard_prot_settle(h, b.tr, 1, 0, b.w, st),
        "next_table": lambda: lib.density_b200_shard_prot_next(h, b.w, 1, b.t, st),
        "next": lambda: lib.density_b200_shard_prot_next(h, b.w, 1, None, st),
        "finish": lambda: lib.density_b200_shard_prot_finish(h, b.o, b.cap, b.sz, b.sm, st),
        "status": lambda: lib.density_b200_shard_prot_status(h, status),
    }


# stage -> the calls that reach it from a new shard
CHAM_STAGES = {
    "new": [],
    "phase1": ["phase1"],
    "phase2": ["phase1", "phase2"],
    "flags": ["prot_phase1"],
    "transfer": ["prot_phase1", "transfer"],
    "settled": ["prot_phase1", "transfer", "settle"],
    "flags_round1": ["prot_phase1", "transfer", "settle", "next_table"],
    "committed": ["prot_phase1", "transfer", "settle", "next"],
    "finished": ["prot_phase1", "transfer", "settle", "next", "finish"],
    "phase1_after_prot": ["prot_phase1", "transfer", "phase1"],
}
# entry -> the stages it may follow
CHAM_ALLOWED = {
    "phase1": set(CHAM_STAGES), "prot_phase1": set(CHAM_STAGES),
    "phase2": {"phase1", "phase2", "phase1_after_prot"},
    "transfer": {"flags", "flags_round1"},
    "settle": {"transfer"},
    "next_table": {"settled"}, "next": {"settled"},
    "finish": {"committed"},
    "status": {"committed", "finished"},
}


@pytest.mark.parametrize("stage", list(CHAM_STAGES))
def test_chameleon_order(torch_cuda, lib, stage):
    torch, st = torch_cuda, _stream(torch_cuda)
    b = Bufs(torch, "chameleon", text(16 * 1024 + 5))
    for entry, allowed in CHAM_ALLOWED.items():
        h = lib.density_b200_shard_create()
        calls = cham_entries(lib, h, b, st)
        for step in CHAM_STAGES[stage]:
            assert calls[step]() == 0, (stage, step, lib.density_b200_last_error())
        if stage in allowed:
            assert calls[entry]() == 0, (stage, entry, lib.density_b200_last_error())
        else:
            refused(lib, calls[entry])
        torch.cuda.synchronize()
        lib.density_b200_shard_destroy(h)


def test_chameleon_round_budget(torch_cuda, lib, budget):
    torch, st = torch_cuda, _stream(torch_cuda)
    b = Bufs(torch, "chameleon", text(16 * 1024 + 5))
    budget(2)
    h = lib.density_b200_shard_create()
    calls = cham_entries(lib, h, b, st)
    for step in ["prot_phase1", "transfer", "settle", "next_table", "transfer", "settle"]:
        assert calls[step]() == 0
    refused(lib, calls["next_table"])          # round + 1 == budget
    assert calls["next"]() == 0 and calls["finish"]() == 0
    torch.cuda.synchronize()
    lib.density_b200_shard_destroy(h)


# ---- the Cheetah / Lion shard -------------------------------------------------------------------------------------------------------
def cl_entries(lib, h, b, st):
    status = (ctypes.c_uint32 * 20)()
    return {
        "phase1": lambda: lib.density_b200_cl_shard_phase1(h, b.i, b.n, 1, None, b.t, st),
        "phase2": lambda: lib.density_b200_cl_shard_phase2(h, None, b.t, st),
        "phase3": lambda: lib.density_b200_cl_shard_phase3(h, None, b.o, b.cap, b.sz, b.sm, st),
        "prot_phase1": lambda: lib.density_b200_cl_shard_prot_phase1(h, b.i, b.n, 0, 1, b.w, st),
        "p": lambda: lib.density_b200_cl_shard_prot_p(h, b.w, 1, 0, b.t, st),
        "c": lambda: lib.density_b200_cl_shard_prot_c(h, b.c, b.t, st),
        "transfer": lambda: lib.density_b200_cl_shard_prot_transfer(h, b.c, b.tr, st),
        "settle": lambda: lib.density_b200_cl_shard_prot_settle(h, b.tr, 1, 0, b.w, st),
        "next": lambda: lib.density_b200_cl_shard_prot_next(h, b.w, 1, st),
        "finish": lambda: lib.density_b200_cl_shard_prot_finish(h, b.o, b.cap, b.sz, b.sm, st),
        "status": lambda: lib.density_b200_cl_shard_prot_status(h, status),
    }


ROUND = ["p", "c", "transfer", "settle", "next"]
CL_STAGES = {
    "new": [],
    "phase1": ["phase1"],
    "phase2": ["phase1", "phase2"],
    "phase3": ["phase1", "phase2", "phase3"],
    "ready": ["prot_phase1"],
    "p": ["prot_phase1", "p"],
    "c": ["prot_phase1", "p", "c"],
    "transfer": ["prot_phase1", "p", "c", "transfer"],
    "settled": ["prot_phase1", "p", "c", "transfer", "settle"],
    "ready_round1": ["prot_phase1"] + ROUND,
    "p_round1": ["prot_phase1"] + ROUND + ["p"],
    "settled_round1": ["prot_phase1"] + ROUND + ["p", "c", "transfer", "settle"],
    "finished": ["prot_phase1"] + ROUND + ["finish"],
    "phase1_after_prot": ["prot_phase1"] + ROUND + ["phase1"],
}
CL_ALLOWED = {
    "phase1": set(CL_STAGES), "prot_phase1": set(CL_STAGES),
    "phase2": {"phase1", "phase1_after_prot"},
    "phase3": {"phase2"},
    "p": {"ready", "ready_round1"},
    "c": {"p", "p_round1"},
    "transfer": {"c"},
    "settle": {"transfer"},
    "next": {"settled", "settled_round1"},
    "finish": {"ready_round1"},
    "status": {"ready_round1", "p_round1", "settled_round1", "finished"},
}


@pytest.mark.parametrize("alg", ["cheetah", "lion"])
@pytest.mark.parametrize("stage", list(CL_STAGES))
def test_cl_order(torch_cuda, lib, alg, stage):
    torch, st = torch_cuda, _stream(torch_cuda)
    b = Bufs(torch, alg, text(16 * 1024 + 5))
    for entry, allowed in CL_ALLOWED.items():
        h = lib.density_b200_cl_shard_create(ALG_ID[alg])
        calls = cl_entries(lib, h, b, st)
        for step in CL_STAGES[stage]:
            assert calls[step]() == 0, (stage, step, lib.density_b200_last_error())
        if stage in allowed:
            assert calls[entry]() == 0, (stage, entry, lib.density_b200_last_error())
        else:
            refused(lib, calls[entry])
        torch.cuda.synchronize()
        lib.density_b200_cl_shard_destroy(h)


@pytest.mark.parametrize("alg", ["cheetah", "lion"])
def test_cl_round_budget(torch_cuda, lib, budget, alg):
    torch, st = torch_cuda, _stream(torch_cuda)
    b = Bufs(torch, alg, text(16 * 1024 + 5))
    budget(1)
    h = lib.density_b200_cl_shard_create(ALG_ID[alg])
    calls = cl_entries(lib, h, b, st)
    for step in ["prot_phase1"] + ROUND:
        assert calls[step]() == 0
    refused(lib, calls["p"])                   # round == budget
    assert calls["finish"]() == 0
    torch.cuda.synchronize()
    lib.density_b200_cl_shard_destroy(h)


# ---- alignment and NULLs ------------------------------------------------------------------------------------------------------------
def test_chameleon_shard_args(torch_cuda, lib):
    torch, st = torch_cuda, _stream(torch_cuda)
    b = Bufs(torch, "chameleon", text(64 * 1024 + 5))
    i, o, t, c, w, tr, sz, sm, fl = b.i, b.o, b.t, b.c, b.w, b.tr, b.sz, b.sm, b.fl
    refused(lib, lambda: lib.density_b200_table_init(t + 2, st), lambda: lib.density_b200_table_init(None, st),
            lambda: lib.density_b200_table_fold(t + 2, c, st), lambda: lib.density_b200_table_fold(t, c + 2, st),
            lambda: lib.density_b200_table_fold(None, c, st), lambda: lib.density_b200_table_fold(t, None, st))
    assert lib.density_b200_table_init(c, st) == 0 and lib.density_b200_table_fold(c, t, st) == 0
    h = lib.density_b200_shard_create()
    ph1 = lambda i, t: lib.density_b200_shard_phase1(h, i, b.n, 1, t, st)
    refused(lib, lambda: ph1(i + 2, t), lambda: ph1(i, t + 2), lambda: ph1(i, None), lambda: ph1(None, t))
    assert ph1(i, t) == 0
    ph2 = lambda c, o, sz, fl: lib.density_b200_shard_phase2(h, c, o, b.cap, sz, fl, st)
    refused(lib, lambda: ph2(c + 2, o, sz, fl), lambda: ph2(None, o + 1, sz, fl), lambda: ph2(None, o, sz + 4, fl),
            lambda: ph2(None, o, None, fl), lambda: ph2(None, o, sz, fl + 2))
    b.flags.fill_(1)
    assert ph2(None, o, sz, fl) == 0
    assert b.encoded(torch) and int(b.flags[0].item()) == 0
    lib.density_b200_shard_destroy(h)

    b = Bufs(torch, "chameleon", with_noise(64 * 1024 + 5))
    i, o, t, w, tr, sz, sm = b.i, b.o, b.t, b.w, b.tr, b.sz, b.sm
    h = lib.density_b200_shard_create()
    pp1 = lambda i, t: lib.density_b200_shard_prot_phase1(h, i, b.n, 0, 1, t, st)
    refused(lib, lambda: pp1(i + 2, t), lambda: pp1(i, t + 2), lambda: pp1(i, None))
    assert pp1(i, t) == 0
    for k in range(lib.density_b200_prot_round_budget()):
        if k > 0:
            assert lib.density_b200_shard_prot_next(h, w, 1, t, st) == 0
        tra = lambda c, x: lib.density_b200_shard_prot_transfer(h, c, x, st)
        se = lambda x, y: lib.density_b200_shard_prot_settle(h, x, 1, 0, y, st)
        if k == 0:
            refused(lib, lambda: tra(b.c + 2, tr), lambda: tra(None, tr + 2), lambda: tra(None, None))
        assert tra(None, tr) == 0
        if k == 0:
            refused(lib, lambda: se(tr + 2, w), lambda: se(tr, w + 2), lambda: se(None, w), lambda: se(tr, None))
        assert se(tr, w) == 0
        if k == 0:
            nx = lambda x, y: lib.density_b200_shard_prot_next(h, x, 1, y, st)
            refused(lib, lambda: nx(w + 2, t), lambda: nx(w, t + 2), lambda: nx(None, t))
    assert lib.density_b200_shard_prot_next(h, w, 1, None, st) == 0
    fin = lambda o, sz, sm: lib.density_b200_shard_prot_finish(h, o, b.cap, sz, sm, st)
    refused(lib, lambda: fin(o + 1, sz, sm), lambda: fin(o, sz + 4, sm), lambda: fin(o, sz, sm + 2), lambda: fin(o, None, sm),
            lambda: fin(o, sz, None), lambda: fin(None, sz, sm))
    assert fin(o, sz, sm) == 0
    assert b.encoded(torch) and int(b.seam[2].item()) == 0
    lib.density_b200_shard_destroy(h)


@pytest.mark.parametrize("alg", ["cheetah", "lion"])
def test_cl_shard_args(torch_cuda, lib, alg):
    torch, st = torch_cuda, _stream(torch_cuda)
    from density_b200 import sharded as S
    a = ALG_ID[alg]
    b = Bufs(torch, alg, text(64 * 1024 + 5))
    i, o, t, c, w, tr, sz, sm = b.i, b.o, b.t, b.c, b.w, b.tr, b.sz, b.sm
    for kind in (S.CL_TABLE_P, S.CL_TABLE_C):
        refused(lib, lambda: lib.density_b200_cl_table_init(a, kind, t + 2, st),
                lambda: lib.density_b200_cl_table_fold(a, kind, t + 2, c, st), lambda: lib.density_b200_cl_table_fold(a, kind, t, c + 2, st))
        assert lib.density_b200_cl_table_init(a, kind, c, st) == 0 and lib.density_b200_cl_table_fold(a, kind, c, t, st) == 0
    h = lib.density_b200_cl_shard_create(a)
    ph1 = lambda i, q, t: lib.density_b200_cl_shard_phase1(h, i, b.n, 1, q, t, st)
    refused(lib, lambda: ph1(i + 2, None, t), lambda: ph1(i, w + 2, t), lambda: ph1(i, None, t + 2), lambda: ph1(i, None, None))
    assert ph1(i, None, t) == 0
    ph2 = lambda c, t: lib.density_b200_cl_shard_phase2(h, c, t, st)
    refused(lib, lambda: ph2(c + 2, t), lambda: ph2(None, t + 2), lambda: ph2(None, None))
    assert ph2(None, t) == 0
    ph3 = lambda c, o, sz, sm: lib.density_b200_cl_shard_phase3(h, c, o, b.cap, sz, sm, st)
    refused(lib, lambda: ph3(c + 2, o, sz, sm), lambda: ph3(None, o + 1, sz, sm), lambda: ph3(None, o, sz + 4, sm),
            lambda: ph3(None, o, sz, sm + 2), lambda: ph3(None, o, None, sm), lambda: ph3(None, o, sz, None))
    assert ph3(None, o, sz, sm) == 0
    assert b.encoded(torch) and int(b.seam[2].item()) == 0
    lib.density_b200_cl_shard_destroy(h)

    b = Bufs(torch, alg, with_noise(64 * 1024 + 5))
    i, o, w, tr, sz, sm = b.i, b.o, b.w, b.tr, b.sz, b.sm
    tp = torch.zeros((1, lib.density_b200_cl_table_words(a, S.CL_TABLE_P)), dtype=torch.int32, device="cuda")
    tc = torch.zeros((1, lib.density_b200_cl_table_words(a, S.CL_TABLE_C)), dtype=torch.int32, device="cuda")
    h = lib.density_b200_cl_shard_create(a)
    pp1 = lambda i, w: lib.density_b200_cl_shard_prot_phase1(h, i, b.n, 0, 1, w, st)
    refused(lib, lambda: pp1(i + 2, w), lambda: pp1(i, w + 2), lambda: pp1(i, None))
    assert pp1(i, w) == 0
    for k in range(lib.density_b200_prot_round_budget()):
        p = lambda x, y: lib.density_b200_cl_shard_prot_p(h, x, 1, 0, y, st)
        if k == 0:
            refused(lib, lambda: p(w + 2, tp.data_ptr()), lambda: p(w, tp.data_ptr() + 2))
        assert p(w, tp.data_ptr()) == 0
        carry_p = S.fold_cl_tables(a, S.CL_TABLE_P, tp, 0).contiguous()
        cc = lambda x, y: lib.density_b200_cl_shard_prot_c(h, x, y, st)
        if k == 0:
            refused(lib, lambda: cc(carry_p.data_ptr() + 2, tc.data_ptr()), lambda: cc(carry_p.data_ptr(), tc.data_ptr() + 2))
        assert cc(carry_p.data_ptr(), tc.data_ptr()) == 0
        carry_c = S.fold_cl_tables(a, S.CL_TABLE_C, tc, 0).contiguous()
        tra = lambda x, y: lib.density_b200_cl_shard_prot_transfer(h, x, y, st)
        if k == 0:
            refused(lib, lambda: tra(carry_c.data_ptr() + 2, tr), lambda: tra(carry_c.data_ptr(), tr + 2))
        assert tra(carry_c.data_ptr(), tr) == 0
        se = lambda x, y: lib.density_b200_cl_shard_prot_settle(h, x, 1, 0, y, st)
        if k == 0:
            refused(lib, lambda: se(tr + 2, w), lambda: se(tr, w + 2))
        assert se(tr, w) == 0
        if k == 0:
            refused(lib, lambda: lib.density_b200_cl_shard_prot_next(h, w + 2, 1, st))
        assert lib.density_b200_cl_shard_prot_next(h, w, 1, st) == 0
    fin = lambda o, sz, sm: lib.density_b200_cl_shard_prot_finish(h, o, b.cap, sz, sm, st)
    refused(lib, lambda: fin(o + 1, sz, sm), lambda: fin(o, sz + 4, sm), lambda: fin(o, sz, sm + 2), lambda: fin(o, None, sm),
            lambda: fin(o, sz, None))
    assert fin(o, sz, sm) == 0
    assert b.encoded(torch) and int(b.seam[2].item()) == 0
    lib.density_b200_cl_shard_destroy(h)


@pytest.mark.parametrize("alg", ["chameleon", "cheetah", "lion"])
@pytest.mark.parametrize("protected", [False, True])
def test_drivers(torch_cuda, lib, alg, protected):
    torch, st = torch_cuda, _stream(torch_cuda)
    from density_b200 import sharded
    b = Bufs(torch, alg, with_noise(64 * 1024 + 5) if protected else text(64 * 1024 + 5))
    enc = sharded.ShardedEncoder(torch.device("cuda"))
    a = ALG_ID[alg]
    if alg == "chameleon":
        fn = lib.density_b200_encode_sharded_protected if protected else lib.density_b200_encode_sharded
        drv = lambda i, o, sz, fl, tot: fn(enc._h, i, b.n, o, b.cap, sz, fl, tot, -1, None, 0, st)
    else:
        fn = lib.density_b200_encode_sharded_cl_protected if protected else lib.density_b200_encode_sharded_cl
        drv = lambda i, o, sz, fl, tot: fn(enc._h, a, i, b.n, o, b.cap, sz, fl, tot, -1, None, 0, st)
    i, o, sz, fl, tot = b.i, b.o, b.sz, b.fl, b.tot
    refused(lib, lambda: drv(i + 2, o, sz, fl, tot), lambda: drv(i, o + 1, sz, fl, tot), lambda: drv(i, o, sz + 4, fl, tot),
            lambda: drv(i, o, sz, fl + 2, tot), lambda: drv(i, o, sz, fl, tot + 4), lambda: drv(None, o, sz, fl, tot),
            lambda: drv(i, None, sz, fl, tot), lambda: drv(i, o, None, fl, tot))
    b.flags.fill_(1)
    assert drv(i, o, sz, fl, tot) == 0, lib.density_b200_last_error()
    assert b.encoded(torch) and int(b.flags[0].item()) == 0 and int(b.total[0].item()) == int(b.size[0].item())
    enc.close()
