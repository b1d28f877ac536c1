"""Sharded Chameleon encode with copy mode (needs an H100: pytest -m gpu). W shards of one input run through the phase API
(density_b200_shard_prot_*) on one device, the exchanges replaced by stacking the tables, transfers and round words and folding the
tables with sharded.fold_tables. Whatever the input -- noise, mixed data, copy runs and penalties pending at the cuts -- the
concatenated pieces equal one chameleon_encode call byte for byte with verdict 0, and the rounds are the single-device rounds."""
import ctypes

import numpy as np
import pytest

import oracle
import protection as P
from conftest import payload

pytestmark = pytest.mark.gpu

MIB = 1 << 20
EARG = 4


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


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def encode_prot_shards(torch, lib, data, cuts, canary=0):
    """Every phase of every shard on one device. Returns (pieces, (flags, total, offsets), per-shard prot_status, round words [k])."""
    from density_b200 import sharded as S
    world, st = len(cuts) - 1, _stream(torch)
    encs = [S.ShardedChameleonEncoder() for _ in range(world)]
    ins = [torch.from_numpy(data[cuts[r]:cuts[r + 1]].copy()).cuda() for r in range(world)]
    tables = torch.empty((world, S.TABLE_ENTRIES), dtype=torch.int32, device="cuda")
    transfers = torch.empty((world, S.PROT_TRANSFER_WORDS), dtype=torch.int32, device="cuda")
    words = torch.empty((world, S.PROT_ROUND_WORDS), dtype=torch.int32, device="cuda")
    for r in range(world):
        rc = lib.density_b200_shard_prot_phase1(encs[r]._h, ins[r].data_ptr(), ins[r].numel(), cuts[r] // 256, int(r == world - 1),
                                                tables[r].data_ptr(), st)
        assert rc == 0, lib.density_b200_last_error()
    rounds = []
    for k in range(lib.density_b200_prot_round_budget()):
        for r in range(world if k else 0):
            assert lib.density_b200_shard_prot_next(encs[r]._h, words.data_ptr(), world, tables[r].data_ptr(), st) == 0
        carries = [S.fold_tables(tables, r).contiguous() for r in range(world)]
        for r in range(world):
            assert lib.density_b200_shard_prot_transfer(encs[r]._h, carries[r].data_ptr(), transfers[r].data_ptr(), st) == 0
        for r in range(world):
            assert lib.density_b200_shard_prot_settle(encs[r]._h, transfers.data_ptr(), world, r, words[r].data_ptr(), st) == 0
        rounds.append(words.clone())
    outs, sizes = [], []
    seams = torch.zeros((world, S.SEAM_WORDS), dtype=torch.int32, device="cuda")
    for r in range(world):
        assert lib.density_b200_shard_prot_next(encs[r]._h, words.data_ptr(), world, None, st) == 0
        cap = lib.chameleon_safe_encode_buffer_size(ins[r].numel())
        d_out = torch.full((cap + 64,), canary, dtype=torch.uint8, device="cuda")
        d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        rc = lib.density_b200_shard_prot_finish(encs[r]._h, d_out.data_ptr(), cap, d_sz.data_ptr(), seams[r].data_ptr(), st)
        assert rc == 0, lib.density_b200_last_error()
        outs.append(d_out); sizes.append(d_sz)
    torch.cuda.synchronize()
    verdict = S.seam_verdict(seams)
    status = [e.prot_status() for e in encs]
    pieces = [outs[r][:int(sizes[r].item())].cpu().numpy() for r in range(world)]
    for r in range(world):
        tail = outs[r][lib.chameleon_safe_encode_buffer_size(ins[r].numel()):]
        assert bool((tail == canary).all()), "written past cap"
    for e in encs:
        e.close()
    return pieces, verdict, status, [w.cpu().numpy() for w in rounds]


def check_equal(torch, lib, data, cuts, want=None):
    pieces, (flags, total, _), status, rounds = encode_prot_shards(torch, lib, data, cuts)
    if want is None:
        want = oracle.encode("chameleon", data)
    assert flags == 0, (cuts, status)
    cat = np.concatenate(pieces)
    assert total == want.size and cat.size == want.size and (cat == want).all(), cuts
    assert all(s["settled"] for s in status)
    return status, rounds


def text(n, first_page=0):
    from density_b200 import synth
    return synth.synth_text(n, first_page=first_page).numpy()


def cuts_at(n, *blocks):
    return [0] + [b * 256 for b in blocks] + [n]


def test_noise_mixed_and_text(torch_cuda, lib):
    from density_b200 import synth
    for data in (payload("random", 3 * MIB + 77, 1), synth.synth_mixed(4 * MIB).numpy(), text(3 * MIB + 3)):
        n = data.size
        for cuts in (cuts_at(n, n // 512), cuts_at(n, 1111, 5003, 9999), cuts_at(n, *range(997, n // 256, n // 256 // 7))):
            check_equal(torch_cuda, lib, data, cuts)


def test_noise_bursts_at_and_across_cuts(torch_cuda, lib):
    data = text(2 * MIB)
    rnd = payload("random", 64 * 1024, 7)
    cuts_b = [1000, 2501, 4097, 6000]
    for i, b in enumerate(cuts_b):          # a burst ending at the cut, one straddling it, one starting at it, one of 3 blocks across
        lo = [b * 256 - 2048, b * 256 - 1024, b * 256, b * 256 - 512][i]
        ln = [2048, 2048, 4096, 768][i]
        data[lo:lo + ln] = rnd[i * 8192:i * 8192 + ln]
    check_equal(torch_cuda, lib, data, cuts_at(data.size, *cuts_b))


def test_every_seam_state_lands_on_a_cut(torch_cuda, lib):
    """The builders of the Cheetah / Lion seam test, for Chameleon: the first shard ends in penalty 0 with start 2..6, previous_incompressible
    0 / 1, after an encoded R, or with a penalty pending; the next shard starts with R or Z. None is refused here."""
    from test_gpu_protection import _shard_cases
    n = 0
    for end, nxt, cut, bld in _shard_cases("chameleon"):
        data, _ = bld.realize()
        check_equal(torch_cuda, lib, data, [0, cut, data.size])
        n += 1
    assert n >= 20


def test_every_reachable_state_and_phase_on_a_cut(torch_cuda, lib):
    """Every reachable (penalty, start, previous_incompressible, counter % 16) in front of a cut, so at every counter phase (cuts are
    256-byte aligned, not 16-block aligned), several states per input (one cut each)."""
    states = sorted(P.reachable_states())
    for i in range(0, len(states), 8):
        bld = P.Builder("chameleon", 33 + i)
        cuts = [0]
        for st in states[i:i + 8]:
            bld.add("Z" * 40)
            b = next(b for b in range(bld.n + 1, bld.n + 2000) if b % 16 == st[3] and len(P.word_to(st[:3], b)) <= b - bld.n)
            bld.place(b, st[:3], "cut")
            cuts.append(b)
            bld.recover()
        bld.add("Z" * 20)
        data, _ = bld.realize()
        check_equal(torch_cuda, lib, data, [c * 256 for c in cuts] + [data.size])


def test_small_and_empty_shards_and_a_ragged_tail(torch_cuda, lib):
    bld = P.Builder("chameleon", 5)
    bld.add("Z" * 50 + "RR" + "Z" * 3 + "R" * 9 + "Z" * 40 + "RRZRRZ" + "Z" * 30)
    data, _ = bld.realize()
    for tail in (1, 2, 3):
        d = np.concatenate([data, payload("random", 256 + tail, tail)])
        n = d.size
        nb = n // 256
        for cuts in ([0, 0, 51 * 256, 52 * 256, 52 * 256, 60 * 256, n],       # empty shards, a cut right after the first block of a pair
                     [0, 56 * 256, 57 * 256, 58 * 256, nb * 256, n],           # inside a copy run, 1-block shards, the tail alone
                     [0, 0, 53 * 256, nb * 256, n]):                            # an empty first shard
            check_equal(torch_cuda, lib, d, cuts)


def _feedback_input():
    """The same incompressible blob in shard 0 and shard 2: shard 2's hits on it depend on whether shard 0 copied it (copy-mode blocks
    never reach the dictionary), so the copy decisions feed each other across the shards through the dictionary."""
    t = text(MIB)
    blob = payload("random", 40 * 256, 9)
    return np.concatenate([t[:100 * 256], blob, t[100 * 256:600 * 256], blob, t[600 * 256:]])


def test_copy_decisions_feed_each_other_across_shards(torch_cuda, lib):
    data = _feedback_input()
    status, rounds = check_equal(torch_cuda, lib, data, cuts_at(data.size, 300, 620, 900))
    assert status[0]["rounds"] > 1 and all(s["rounds"] == status[0]["rounds"] for s in status)
    assert sum(s["changed"][1] for s in status) > 0


def test_rounds_equal_the_single_device_rounds(torch_cuda, lib):
    """Per round, the changed blocks summed over the shards equal density_b200_prot_debug after a single-device path-4 encode of the
    whole input: path 4 numbers rounds 0..4, then reuses slots 8..15 for round 5 on."""
    import torch
    from density_b200 import synth
    for data, cuts in ((_feedback_input(), (300, 620, 900)), (synth.synth_mixed(4 * MIB).numpy(), (1001, 7777, 12000))):
        status, _ = check_equal(torch, lib, data, cuts_at(data.size, *cuts))
        d_in = torch.from_numpy(data.copy()).cuda()
        d_out = torch.zeros(lib.chameleon_safe_encode_buffer_size(data.size), dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        assert lib.density_b200_encode_device_path(0, d_in.data_ptr(), data.size, d_out.data_ptr(), d_out.numel(), d_sz.data_ptr(),
                                                   _stream(torch), 4) == 0
        torch.cuda.synchronize()
        dbg = (ctypes.c_uint64 * 32)()
        assert lib.density_b200_prot_debug(dbg) == 0
        used = status[0]["rounds"]
        assert 1 <= used <= 12
        slot = lambda k: k if k < 5 else k + 3
        for k in range(used):
            assert sum(s["changed"][k] for s in status) == dbg[2 * slot(k) + 1], (k, used)
        # both settled in the same round: no change in it, and the single device ran no round after it
        assert sum(s["changed"][used - 1] for s in status) == 0
        assert dbg[2 * slot(used) + 1] == 0 and dbg[2 * slot(used)] == 2 ** 64 - 1, (used, list(dbg))


def test_budget_below_what_the_input_needs_is_refused(torch_cuda, lib, budget):
    data = _feedback_input()
    cuts = cuts_at(data.size, 300, 620, 900)
    status, _ = check_equal(torch_cuda, lib, data, cuts)
    lib.density_b200_test_set_prot_rounds(status[0]["rounds"] - 1)
    pieces, (flags, total, _), status, _ = encode_prot_shards(torch_cuda, lib, data, cuts, canary=0xA5)
    assert flags != 0 and total == 0 and all(p.size == 0 for p in pieces)
    assert not any(s["settled"] for s in status)


def test_quiet_text_equals_the_quiet_path(torch_cuda, lib):
    """On quiet input the pieces equal those of density_b200_shard_phase1 / 2, and the map settles in round 0."""
    from density_b200 import sharded as S
    torch = torch_cuda
    data = text(4 * MIB)
    cuts = cuts_at(data.size, 4000, 8192, 12001)
    pieces, (flags, _, _), status, _ = encode_prot_shards(torch, lib, data, cuts)
    assert flags == 0 and all(s["rounds"] == 1 for s in status)
    world, st = len(cuts) - 1, _stream(torch)
    encs = [S.ShardedChameleonEncoder() for _ in range(world)]
    ins = [torch.from_numpy(data[cuts[r]:cuts[r + 1]].copy()).cuda() for r in range(world)]
    tables = torch.empty((world, S.TABLE_ENTRIES), dtype=torch.int32, device="cuda")
    for r in range(world):
        assert lib.density_b200_shard_phase1(encs[r]._h, ins[r].data_ptr(), ins[r].numel(), int(r == world - 1), tables[r].data_ptr(), st) == 0
    fl = torch.zeros(world, dtype=torch.int32, device="cuda")
    for r in range(world):
        carry = S.fold_tables(tables, r).contiguous() if r else None
        d_out = torch.zeros(lib.chameleon_safe_encode_buffer_size(ins[r].numel()), dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        assert lib.density_b200_shard_phase2(encs[r]._h, carry.data_ptr() if carry is not None else None, d_out.data_ptr(), d_out.numel(),
                                             d_sz.data_ptr(), fl[r].data_ptr(), st) == 0
        torch.cuda.synchronize()
        assert (d_out[:int(d_sz.item())].cpu().numpy() == pieces[r]).all() and d_sz.item() == pieces[r].size
    assert int(fl.sum().item()) == 0
    for e in encs:
        e.close()


def test_encode_device_launch_count_is_unchanged(torch_cuda, lib):
    """encode_device (path 0) keeps its kernels on quiet and on non-quiet input alike: the flag pass; carry scan, resolve and sizes;
    rounds 0..4 of the copy-map iteration (prot_iterate, and before rounds 1..4 the flag pass, carry scan and resolve); the in-order
    kernel, the sizes under the copy map, the two scan kernels and the emit."""
    import torch
    from density_b200 import synth
    for data in (text(2 * MIB), synth.synth_mixed(2 * MIB).numpy()):
        d_in = torch.from_numpy(data.copy()).cuda()
        d_out = torch.zeros(lib.chameleon_safe_encode_buffer_size(data.size), dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        before = lib.density_b200_kernel_launches()
        assert lib.density_b200_encode_device(0, d_in.data_ptr(), data.size, d_out.data_ptr(), d_out.numel(), d_sz.data_ptr(), _stream(torch)) == 0
        torch.cuda.synchronize()
        assert lib.density_b200_kernel_launches() - before == 1 + 3 + (1 + 4 * 4) + 5
        assert (d_out[:int(d_sz.item())].cpu().numpy() == oracle.encode("chameleon", data)).all()


def test_quiet_phase1_voids_the_copy_map_phases(torch_cuda, lib):
    """The quiet phase 1 takes over the handle's workspace: the copy-map phases on the same handle start over with prot_phase1."""
    from density_b200 import sharded as S
    torch = torch_cuda
    st = _stream(torch)
    enc = S.ShardedChameleonEncoder()
    d_in = torch.from_numpy(text(64 * 1024)).cuda()
    tab = torch.empty(S.TABLE_ENTRIES, dtype=torch.int32, device="cuda")
    tr = torch.empty(S.PROT_TRANSFER_WORDS, dtype=torch.int32, device="cuda")
    assert lib.density_b200_shard_prot_phase1(enc._h, d_in.data_ptr(), d_in.numel(), 0, 1, tab.data_ptr(), st) == 0
    assert lib.density_b200_shard_phase1(enc._h, d_in.data_ptr(), d_in.numel(), 1, tab.data_ptr(), st) == 0
    torch.cuda.synchronize()
    before = lib.density_b200_kernel_launches()
    assert lib.density_b200_shard_prot_transfer(enc._h, None, tr.data_ptr(), st) == EARG
    assert lib.density_b200_kernel_launches() == before
    torch.cuda.synchronize()
    enc.close()


def test_encode_sharded_protected_bad_arguments_before_any_collective(torch_cuda, lib):
    from density_b200 import sharded as S
    torch = torch_cuda
    enc = S.ShardedEncoder(torch.device("cuda"))
    d_in = torch.from_numpy(text(64 * 1024)).cuda()
    cap = lib.chameleon_safe_encode_buffer_size(d_in.numel())
    d_out = torch.zeros(cap + 8, dtype=torch.uint8, device="cuda")
    words = torch.zeros(4, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    before = lib.density_b200_kernel_launches()
    fn = lib.density_b200_encode_sharded_protected
    st = _stream(torch)
    for sz, fl, tot in ((words.data_ptr() + 4, words[1].data_ptr(), words[2].data_ptr()),     # misaligned size
                        (words.data_ptr(), words[1].data_ptr() + 2, words[2].data_ptr()),     # misaligned flags
                        (words.data_ptr(), words[1].data_ptr(), words[2].data_ptr() + 4)):    # misaligned total
        assert fn(enc._h, d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), cap, sz, fl, tot, -1, None, 0, st) == EARG
    assert lib.density_b200_kernel_launches() == before
    enc.close()


def test_encode_sharded_protected_world1_equals_encode_device(torch_cuda, lib):
    import density_b200
    from density_b200 import sharded as S, synth
    torch = torch_cuda
    enc = S.ShardedEncoder(torch.device("cuda"))
    for data in (synth.synth_mixed(3 * MIB + 5).numpy(), payload("random", MIB, 4), text(MIB)):
        d_in = torch.from_numpy(data.copy()).cuda()
        cap = lib.chameleon_safe_encode_buffer_size(data.size)
        want = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        w_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        density_b200.encode_device("chameleon", d_in, want, w_sz)
        d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        d_gather = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_fl = torch.ones(1, dtype=torch.int32, device="cuda")
        enc.encode_protected(d_in, d_out, d_sz, d_fl, gather_root=0, d_gather=d_gather)
        torch.cuda.synchronize()
        n = int(w_sz.item())
        assert int(d_fl.item()) == 0 and int(d_sz.item()) == n == int(enc.d_total.item())
        assert torch.equal(d_out[:n], want[:n]) and torch.equal(d_gather[:n], want[:n])
        assert all(t >= 0 for t in enc.profile())
    enc.close()


def test_python_phase_driver_world1(torch_cuda, lib):
    from density_b200 import sharded as S, synth
    torch = torch_cuda
    data = synth.synth_mixed(2 * MIB).numpy()
    d_in = torch.from_numpy(data.copy()).cuda()
    d_out = torch.zeros(lib.chameleon_safe_encode_buffer_size(data.size), dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    enc = S.ShardedChameleonEncoder()
    flags, total, _ = enc.encode_protected(d_in, d_out, d_sz)
    want = oracle.encode("chameleon", data)
    assert flags == 0 and total == want.size and (d_out[:total].cpu().numpy() == want).all()
    assert enc.prot_status()["settled"] == 1 and enc.prot_status()["in_state"] == (0, 1, 0)
    enc.close()


def test_bad_arguments_enqueue_nothing(torch_cuda, lib):
    from density_b200 import sharded as S
    torch = torch_cuda
    st = _stream(torch)
    enc = S.ShardedChameleonEncoder()
    d_in = torch.from_numpy(text(64 * 1024)).cuda()
    tab = torch.empty(S.TABLE_ENTRIES + 1, dtype=torch.int32, device="cuda")
    tr = torch.empty(S.PROT_TRANSFER_WORDS, dtype=torch.int32, device="cuda")
    w = torch.empty(S.PROT_ROUND_WORDS, dtype=torch.int32, device="cuda")
    out = torch.empty(lib.chameleon_safe_encode_buffer_size(d_in.numel()) + 2, dtype=torch.uint8, device="cuda")
    sz = torch.empty(1, dtype=torch.int64, device="cuda")
    seam = torch.empty(8, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    before = lib.density_b200_kernel_launches()
    h = enc._h
    assert lib.density_b200_shard_prot_transfer(h, None, tr.data_ptr(), st) == EARG                                   # before phase 1
    assert lib.density_b200_shard_prot_phase1(h, d_in.data_ptr() + 1, 4096, 0, 1, tab.data_ptr(), st) == EARG         # misaligned input
    assert lib.density_b200_shard_prot_phase1(h, d_in.data_ptr(), 4096, 0, 1, tab.data_ptr() + 2, st) == EARG         # misaligned table
    assert lib.density_b200_shard_prot_phase1(h, d_in.data_ptr(), 1000, 0, 0, tab.data_ptr(), st) == EARG             # non-final, not 256k
    assert lib.density_b200_kernel_launches() == before
    assert lib.density_b200_shard_prot_phase1(h, d_in.data_ptr(), d_in.numel(), 0, 1, tab.data_ptr(), st) == 0
    before = lib.density_b200_kernel_launches()
    assert lib.density_b200_shard_prot_settle(h, tr.data_ptr(), 1, 0, w.data_ptr(), st) == EARG                      # before transfer
    assert lib.density_b200_shard_prot_next(h, w.data_ptr(), 1, tab.data_ptr(), st) == EARG                          # before settle
    assert lib.density_b200_shard_prot_finish(h, out.data_ptr(), out.numel(), sz.data_ptr(), seam.data_ptr(), st) == EARG
    assert lib.density_b200_shard_prot_transfer(h, None, tr.data_ptr() + 1, st) == EARG                               # misaligned
    assert lib.density_b200_kernel_launches() == before
    assert lib.density_b200_shard_prot_transfer(h, None, tr.data_ptr(), st) == 0
    assert lib.density_b200_shard_prot_transfer(h, None, tr.data_ptr(), st) == EARG                                   # twice
    assert lib.density_b200_shard_prot_settle(h, tr.data_ptr(), 1, 1, w.data_ptr(), st) == EARG                      # rank >= world
    assert lib.density_b200_shard_prot_settle(h, tr.data_ptr(), 1, 0, w.data_ptr(), st) == 0
    before = lib.density_b200_kernel_launches()
    assert lib.density_b200_shard_prot_finish(h, out.data_ptr(), out.numel(), sz.data_ptr(), seam.data_ptr(), st) == EARG  # not committed
    assert lib.density_b200_shard_prot_next(h, w.data_ptr(), 1, None, st) == 0
    assert lib.density_b200_kernel_launches() > before
    before = lib.density_b200_kernel_launches()
    assert lib.density_b200_shard_prot_finish(h, out.data_ptr() + 1, out.numel(), sz.data_ptr(), seam.data_ptr(), st) == EARG  # misaligned
    assert lib.density_b200_kernel_launches() == before
    assert lib.density_b200_shard_prot_finish(h, out.data_ptr(), out.numel(), sz.data_ptr(), seam.data_ptr(), st) == 0
    torch.cuda.synchronize()
    enc.close()


def _nccl_worker(rank, world, port, data, cuts, q):
    import os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import density_b200
    from density_b200 import sharded
    enc = sharded.ShardedEncoder(dev)
    d_in = torch.from_numpy(data[cuts[rank]:cuts[rank + 1]].copy()).to(dev)
    cap = density_b200.Chameleon.safe_encode_buffer_size(d_in.numel())
    d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    enc.encode_protected(d_in, d_out, d_sz, d_fl)
    torch.cuda.synchronize()
    q.put((rank, int(d_fl.item()), d_out[:int(d_sz.item())].cpu().numpy()))
    dist.barrier()
    enc.close()
    dist.destroy_process_group()


def test_encode_sharded_protected_two_ranks_nccl_equals_oracle(torch_cuda):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    data = _feedback_input()
    cuts = cuts_at(data.size, 450)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, 29733, data, cuts, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict((r, (fl, piece)) for r, fl, piece in (q.get(timeout=600) for _ in range(2)))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    want = oracle.encode("chameleon", data)
    assert all(got[r][0] == 0 for r in range(2))
    cat = np.concatenate([got[r][1] for r in range(2)])
    assert cat.size == want.size and (cat == want).all()
