"""Sharded Cheetah and Lion encode with copy mode on every shard (needs an H100: pytest -m gpu). W shards of one input run through the
phase API (density_b200_cl_shard_prot_*) on one device, the exchanges replaced by stacking the round words, tables and transfers and
folding the tables with sharded.fold_cl_tables. Whatever the input -- noise, mixed data, copy runs and penalties pending at the cuts, an
empty first shard -- the concatenated pieces equal one cheetah_encode / lion_encode call byte for byte with verdict 0."""
import ctypes

import numpy as np
import pytest

import oracle
import protection as P
from conftest import payload

pytestmark = pytest.mark.gpu

MIB = 1 << 20
EARG = 4
ALGS = ["cheetah", "lion"]
ALG_ID = {"cheetah": 1, "lion": 2}


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
    yield lib
    lib.density_b200_test_set_prot_rounds(0)     # back to the default budget


@pytest.fixture
def stage_rounds(lib):
    yield lib
    lib.density_b200_test_set_stage_rounds(7)     # back to every round of every stage


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def encode_shards(torch, lib, alg, data, cuts, canary=0):
    """Every phase of every shard on one device. Returns (pieces, (flags, total, offsets), per-shard prot_status)."""
    from density_b200 import sharded as S
    world, st = len(cuts) - 1, _stream(torch)
    a = ALG_ID[alg]
    encs = [S.ShardedCLEncoder(alg) for _ in range(world)]
    ins = [torch.from_numpy(data[cuts[r]:cuts[r + 1]].copy()).cuda() for r in range(world)]
    wp, wc = encs[0].words_p, encs[0].words_c
    words = torch.zeros((world, S.CL_PROT_ROUND_WORDS), dtype=torch.int32, device="cuda")
    tp = torch.zeros((world, wp), dtype=torch.int32, device="cuda")
    tc = torch.zeros((world, wc), dtype=torch.int32, device="cuda")
    transfers = torch.zeros((world, S.PROT_TRANSFER_WORDS), dtype=torch.int32, device="cuda")
    for r in range(world):
        rc = lib.density_b200_cl_shard_prot_phase1(encs[r]._h, ins[r].data_ptr() if ins[r].numel() else None, ins[r].numel(), cuts[r],
                                                   int(r == world - 1), words[r].data_ptr(), st)
        assert rc == 0, lib.density_b200_last_error()
    for _ in range(lib.density_b200_prot_round_budget()):
        for r in range(world):
            assert lib.density_b200_cl_shard_prot_p(encs[r]._h, words.data_ptr(), world, r, tp[r].data_ptr(), st) == 0
        carries = [S.fold_cl_tables(a, S.CL_TABLE_P, tp, r).contiguous() for r in range(world)]
        for r in range(world):
            assert lib.density_b200_cl_shard_prot_c(encs[r]._h, carries[r].data_ptr(), tc[r].data_ptr(), st) == 0
        carries = [S.fold_cl_tables(a, S.CL_TABLE_C, tc, r).contiguous() for r in range(world)]
        for r in range(world):
            assert lib.density_b200_cl_shard_prot_transfer(encs[r]._h, carries[r].data_ptr(), transfers[r].data_ptr(), st) == 0
        for r in range(world):
            assert lib.density_b200_cl_shard_prot_settle(encs[r]._h, transfers.data_ptr(), world, r, words[r].data_ptr(), st) == 0
        for r in range(world):
            assert lib.density_b200_cl_shard_prot_next(encs[r]._h, words.data_ptr(), world, st) == 0
    safe = getattr(lib, f"{alg}_safe_encode_buffer_size")
    outs, sizes = [], []
    seams = torch.zeros((world, S.SEAM_WORDS), dtype=torch.int32, device="cuda")
    for r in range(world):
        cap = safe(ins[r].numel())
        d_out = torch.full((cap + 64,), canary, dtype=torch.uint8, device="cuda")
        d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        rc = lib.density_b200_cl_shard_prot_finish(encs[r]._h, d_out.data_ptr(), cap, d_sz.data_ptr(), seams[r].data_ptr(), st)
        assert rc == 0, lib.density_b200_last_error()
        outs.append(d_out); sizes.append(d_sz)
    torch.cuda.synchronize()
    verdict = S.seam_verdict(seams)
    status = [e.prot_status() for e in encs]
    pieces = [outs[r][:int(sizes[r].item())].cpu().numpy() for r in range(world)]
    for r in range(world):
        assert bool((outs[r][safe(ins[r].numel()):] == canary).all()), "written past cap"
    for e in encs:
        e.close()
    return pieces, verdict, status


def check_equal(torch, lib, alg, data, cuts, want=None):
    pieces, (flags, total, _), status = encode_shards(torch, lib, alg, data, cuts)
    if want is None:
        want = oracle.encode(alg, data)
    assert flags == 0, (alg, cuts, status)
    cat = np.concatenate(pieces)
    assert total == want.size and cat.size == want.size and (cat == want).all(), (alg, cuts)
    assert all(s["stage_settled"] and s["rounds"] > 0 and not s["esc"] for s in status)
    assert len({s["rounds"] for s in status}) == 1
    return status


def text(n, first_page=0):
    from density_b200 import synth
    return synth.synth_text(n, first_page=first_page).numpy()


def cuts_at(n, *units):
    """cuts at multiples of 256 bytes (units), which are not 16-block aligned for either algorithm unless the unit count is"""
    return [0] + [u * 256 for u in units] + [n]


@pytest.mark.parametrize("alg", ALGS)
def test_noise_mixed_and_text(torch_cuda, lib, alg):
    from density_b200 import synth
    for data in (payload("random", MIB + 77, 1), synth.synth_mixed(2 * MIB).numpy(), text(MIB + 3, first_page=3)):
        n = data.size
        for cuts in (cuts_at(n, n // 512), cuts_at(n, 1111, 2003, 3001), cuts_at(n, *range(397, n // 256, n // 256 // 8))):
            check_equal(torch_cuda, lib, alg, data, cuts)


@pytest.mark.parametrize("alg", ALGS)
def test_noise_bursts_at_and_across_cuts(torch_cuda, lib, alg):
    data = text(2 * MIB, first_page=2)
    rnd = payload("random", 64 * 1024, 7)
    cuts_b = [1000, 2501, 4097, 6000]
    for i, b in enumerate(cuts_b):          # a burst ending at the cut, one straddling it, one starting at it, one across
        lo = [b * 256 - 2048, b * 256 - 1024, b * 256, b * 256 - 512][i]
        ln = [2048, 2048, 4096, 768][i]
        data[lo:lo + ln] = rnd[i * 8192:i * 8192 + ln]
    check_equal(torch_cuda, lib, alg, data, cuts_at(data.size, *cuts_b))


@pytest.mark.parametrize("alg", ALGS)
def test_ragged_shards_empty_shards_and_short_tails(torch_cuda, lib, alg):
    from density_b200 import synth
    mixed = synth.synth_mixed(MIB).numpy()
    rng = np.random.default_rng(5)
    for world in range(2, 10):
        tail = int(rng.integers(1, 200))
        d = np.concatenate([mixed[:(mixed.size // 256 - 1) * 256], payload("random", tail, world)])
        body = d.size // 256
        inner = sorted(int(v) for v in rng.choice(np.arange(1, body), world - 2, replace=False))
        cuts = [0] + [256 * u for u in inner] + [256 * body, d.size]
        check_equal(torch_cuda, lib, alg, d, cuts)
    d = mixed[:200 * 1024 + 3]
    n, nb = d.size, d.size // 256
    for cuts in ([0, 0, 0, 300 * 256, n],                      # an empty first shard (and a second): the stream start on shard 2
                 [0, 100 * 256, 100 * 256, 100 * 256, n],       # empty middle shards
                 [0, 256, 512, 768, 1024, nb * 256, n]):        # 256-byte shards, and a last shard shorter than one block
        check_equal(torch_cuda, lib, alg, d, cuts)


@pytest.mark.parametrize("alg", ALGS)
def test_first_shard_with_the_staged_iteration(torch_cuda, lib, alg):
    """a first shard of more than 2 MiB runs stages A and B of the staged iteration (the first MiB alone, then the whole shard)"""
    data = text(3 * MIB + 5, first_page=4)
    data[2 * MIB + 4096:2 * MIB + 4096 + 64 * 1024] = payload("random", 64 * 1024, 3)
    check_equal(torch_cuda, lib, alg, data, cuts_at(data.size, (5 * MIB // 2) // 256 + 3))


@pytest.mark.parametrize("alg", ALGS)
def test_every_seam_case_is_accepted(torch_cuda, lib, alg):
    """The seam cases of the quiet-only path, which refuses some of them; shard 1's incoming state is the single call's at the cut."""
    from test_gpu_protection import _shard_cases
    n = 0
    for end, nxt, cut, bld in _shard_cases(alg):
        data, _ = bld.realize()
        want = oracle.encode(alg, data)
        status = check_equal(torch_cuda, lib, alg, data, [0, cut, data.size], want)
        tr = P.trace(alg, want, data.size)
        assert status[1]["in_state"] == tuple(tr.state[cut // P.BS[alg]]), (end, nxt)
        n += 1
    assert n >= 20


def _feedback_input():
    """The same incompressible blob in shard 0 and shard 2: shard 2's hits on it depend on whether shard 0 copied it (copy-mode blocks
    never reach the tables), so copy decisions near the end of one shard change the compressibility of blocks in a later one."""
    t = text(MIB, first_page=1)
    blob = payload("random", 40 * 256, 9)
    return np.concatenate([t[:100 * 256], blob, t[100 * 256:600 * 256], blob, t[600 * 256:]])


@pytest.mark.parametrize("alg", ALGS)
def test_copy_decisions_feed_each_other_across_shards(torch_cuda, lib, alg):
    data = _feedback_input()
    status = check_equal(torch_cuda, lib, alg, data, cuts_at(data.size, 137, 300, 620, 900))
    assert status[0]["rounds"] > 1


@pytest.mark.parametrize("alg", ALGS)
def test_budget_too_small_is_refused_without_writes_past_cap(torch_cuda, budget, alg):
    lib = budget
    data = _feedback_input()
    cuts = cuts_at(data.size, 137, 300, 620, 900)
    need = check_equal(torch_cuda, lib, alg, data, cuts)[0]["rounds"]
    lib.density_b200_test_set_prot_rounds(need - 1)
    pieces, (flags, total, _), status = encode_shards(torch_cuda, lib, alg, data, cuts, canary=0xA5)
    assert flags != 0 and total == 0 and all(p.size == 0 for p in pieces)
    assert all(s["rounds"] == 0 for s in status)


@pytest.mark.parametrize("alg", ALGS)
def test_first_shard_whose_stages_do_not_settle_is_refused(torch_cuda, stage_rounds, alg):
    """With every stage of the staged iteration cut to one round (test hook), the first shard's map normally does not settle on mixed
    data (the relaxation inside a round reads other SMs' states as they come, so a round may get further on one run than on another):
    then the whole sharded encode is refused and the first shard emits nothing; when it did settle, the pieces are exact."""
    lib, torch = stage_rounds, torch_cuda
    lib.density_b200_test_set_stage_rounds(1)
    refused = 0
    for seed in (9, 10, 11):
        data = payload("mixed", 4 * MIB + 5, seed)
        pieces, (flags, _, _), status = encode_shards(torch, lib, alg, data, [0, 4 * MIB, data.size], canary=0xA5)
        if status[0]["stage_settled"]:
            assert flags == 0 and (np.concatenate(pieces) == oracle.encode(alg, data)).all()
        else:
            assert flags != 0 and pieces[0].size == 0      # the verdict voids the other pieces
            refused += 1
    assert refused, "every first shard settled: these inputs do not exercise the refusal"


@pytest.mark.parametrize("alg", ALGS)
def test_argument_and_phase_order_errors_enqueue_nothing(torch_cuda, lib, alg):
    torch = torch_cuda
    from density_b200 import sharded as S
    st = _stream(torch)
    e = S.ShardedCLEncoder(alg)
    h = e._h
    d = torch.from_numpy(text(64 * 1024 + 64)).cuda()
    w = torch.zeros(64, dtype=torch.int32, device="cuda")
    t = torch.zeros(e.words_p + e.words_c + 256, dtype=torch.int32, device="cuda")
    out = torch.zeros(2 * d.numel(), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(2, dtype=torch.int64, device="cuda")
    before = lib.density_b200_kernel_launches()
    bad = [
        lambda: lib.density_b200_cl_shard_prot_p(h, w.data_ptr(), 1, 0, t.data_ptr(), st),               # before phase 1
        lambda: lib.density_b200_cl_shard_prot_finish(h, out.data_ptr(), out.numel(), sz.data_ptr(), w.data_ptr(), st),
        lambda: lib.density_b200_cl_shard_prot_phase1(h, d.data_ptr() + 1, 1024, 0, 1, w.data_ptr(), st),   # d_in misaligned
        lambda: lib.density_b200_cl_shard_prot_phase1(h, d.data_ptr(), 1000, 0, 0, w.data_ptr(), st),       # non-final, not 256 * k
        lambda: lib.density_b200_cl_shard_prot_phase1(h, d.data_ptr(), 1024, 100, 1, w.data_ptr(), st),     # offset not 256 * k
    ]
    for f in bad:
        assert f() == EARG
    assert lib.density_b200_kernel_launches() == before
    assert lib.density_b200_cl_shard_prot_phase1(h, d.data_ptr(), d.numel(), 0, 1, w.data_ptr(), st) == 0
    before = lib.density_b200_kernel_launches()
    bad = [
        lambda: lib.density_b200_cl_shard_prot_c(h, t.data_ptr(), t.data_ptr(), st),                         # P first
        lambda: lib.density_b200_cl_shard_prot_settle(h, t.data_ptr(), 1, 0, w.data_ptr(), st),
        lambda: lib.density_b200_cl_shard_prot_next(h, w.data_ptr(), 1, st),
        lambda: lib.density_b200_cl_shard_prot_finish(h, out.data_ptr(), out.numel(), sz.data_ptr(), w.data_ptr(), st),  # no round
        lambda: lib.density_b200_cl_shard_prot_p(h, w.data_ptr() + 2, 1, 0, t.data_ptr(), st),             # words misaligned
        lambda: lib.density_b200_cl_shard_prot_p(h, w.data_ptr(), 1, 1, t.data_ptr(), st),                 # rank >= world
    ]
    for f in bad:
        assert f() == EARG
    assert lib.density_b200_kernel_launches() == before
    assert lib.density_b200_cl_shard_prot_p(h, w.data_ptr(), 1, 0, t.data_ptr(), st) == 0
    before = lib.density_b200_kernel_launches()
    assert lib.density_b200_cl_shard_prot_finish(h, out.data_ptr() + 1, out.numel(), sz.data_ptr(), w.data_ptr(), st) == EARG
    assert lib.density_b200_kernel_launches() == before
    # a quiet phase 1 on the same handle closes the copy-map phases
    assert lib.density_b200_cl_shard_phase1(h, d.data_ptr(), d.numel(), 1, None, t.data_ptr(), st) == 0
    before = lib.density_b200_kernel_launches()
    assert lib.density_b200_cl_shard_prot_c(h, t.data_ptr(), t.data_ptr(), st) == EARG
    assert lib.density_b200_cl_shard_prot_p(h, w.data_ptr(), 1, 0, t.data_ptr(), st) == EARG
    assert lib.density_b200_kernel_launches() == before
    torch.cuda.synchronize()
    e.close()


@pytest.mark.parametrize("alg", ALGS)
def test_world_one_entry_equals_the_single_call_and_decodes(torch_cuda, lib, alg):
    torch = torch_cuda
    from density_b200 import synth
    from density_b200.sharded import ShardedEncoder
    data = synth.synth_mixed(3 * MIB).numpy()[:3 * MIB - 5]
    want = oracle.encode(alg, data)
    enc = ShardedEncoder("cuda")
    d_in = torch.from_numpy(data.copy()).cuda()
    cap = getattr(lib, f"{alg}_safe_encode_buffer_size")(data.size)
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_fl = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    d_g = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    enc.encode_protected(d_in, d_out, d_sz, d_fl, gather_root=0, d_gather=d_g, alg=alg)
    torch.cuda.synchronize()
    assert int(d_fl.item()) == 0 and int(d_sz.item()) == want.size == int(enc.d_total.item())
    got = d_g[:want.size].cpu().numpy()
    assert (got == want).all()
    assert all(x >= 0 for x in enc.profile())
    back = torch.zeros(data.size, dtype=torch.uint8, device="cuda")
    bsz = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.density_b200_decode_device(ALG_ID[alg], d_g.data_ptr(), want.size, back.data_ptr(), back.numel(), bsz.data_ptr(),
                                          _stream(torch)) == 0
    torch.cuda.synchronize()
    assert int(bsz.item()) == data.size and (back.cpu().numpy() == data).all()
    enc.close()
