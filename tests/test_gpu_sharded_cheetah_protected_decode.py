"""Sharded Cheetah decode of streams with copy-mode blocks, through the phase API on one device (needs an H100: pytest -m gpu).

W pieces run density_b200_cheetah_decode_shard_prot_transfer / _prot_phase1, then the quiet path's phase 2, rounds and phase 3, the
exchanges replaced by stacking the transfers, chunk-map and prediction tables and round words and folding the tables with the library's
folds. Whatever the data -- noise, synth_mixed, text with noise bursts at and across the cuts, the seam cases of every automaton state,
copy decisions that feed each other -- every piece of the protected sharded Cheetah encoder, and every slice of one cheetah_encode stream
at the same prefix sums, decodes to its shard byte for byte with verdict 0, and the composed transfers are the in-order automaton of the
stream at every cut."""
import ctypes

import numpy as np
import pytest

import oracle
import protection as P
from conftest import payload, splitmix_bytes

pytestmark = pytest.mark.gpu

MIB = 1 << 20
CANARY = 0xA5
EARG = 4
ALG = "cheetah"
BS = P.BS[ALG]


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


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return t.data_ptr() if t.numel() else None


def decode_prot_pieces(torch, lib, pieces, caps):
    """Every phase of every piece on one device. Returns (flags, total, outs, transfers [W, 3200] as numpy, seam words [W, 8]). Checks
    that nothing is written past cap and pins the launches of the protected steps."""
    from density_b200 import sharded as S
    world, st = len(pieces), _stream(torch)
    wc, wp = lib.density_b200_cheetah_cmap_words(), lib.density_b200_cl_table_words(1, S.CL_TABLE_P)
    hs = [lib.density_b200_cheetah_decode_shard_create() for _ in range(world)]
    ins = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in pieces]
    outs = [torch.full((caps[r] + 64,), CANARY, dtype=torch.uint8, device="cuda") for r in range(world)]
    transfers = torch.full((world, S.DECODE_PROT_TRANSFER_WORDS), -1, dtype=torch.int32, device="cuda")
    tc = torch.zeros((world, wc), dtype=torch.int32, device="cuda")

    def launches(fn, *args):
        before = lib.density_b200_kernel_launches()
        rc = fn(*args)
        assert rc == 0, lib.density_b200_last_error()
        return lib.density_b200_kernel_launches() - before

    for r in range(world):
        n, last = ins[r].numel(), r == world - 1
        k = launches(lib.density_b200_cheetah_decode_shard_prot_transfer, hs[r], _ptr(ins[r]), n, outs[r].data_ptr(), caps[r], int(r == 0),
                     int(last), transfers[r].data_ptr(), st)
        assert k == (3 if n else 1)                      # candidate rows, group rows, head walk
    for r in range(world):
        n, last = ins[r].numel(), r == world - 1
        k = launches(lib.density_b200_cheetah_decode_shard_prot_phase1, hs[r], transfers.data_ptr(), world, r,
                     None if last else tc[r].data_ptr(), st)
        # the seed, 7 boundary kernels on the rows of the transfer, the end of the piece, unpack, chunk-map walk, the export
        assert k == (1 + (7 + 1 + 2 if n else 0) + (0 if last else 1)), (r, k)
    for r in range(world):
        carry = S.fold_cheetah_cmap(tc, r) if r > 0 else None
        assert lib.density_b200_cheetah_decode_shard_phase2(hs[r], carry.data_ptr() if carry is not None else None, st) == 0
    tp = torch.zeros((world, wp), dtype=torch.int32, device="cuda")
    words = torch.zeros((world, 4), dtype=torch.int32, device="cuda")
    for _ in range(lib.density_b200_cheetah_decode_round_budget()):
        for r in range(world):
            assert lib.density_b200_cheetah_decode_shard_round_walk(hs[r], tp[r].data_ptr(), words[r].data_ptr(), st) == 0
        for r in range(world):
            carry = S.fold_cl_tables(ALG, S.CL_TABLE_P, tp, r) if r > 0 else None
            rc = lib.density_b200_cheetah_decode_shard_round_fold(hs[r], carry.data_ptr() if carry is not None else None, words.data_ptr(),
                                                                  world, r, st)
            assert rc == 0, lib.density_b200_last_error()
    seam = torch.zeros((world, 8), dtype=torch.int32, device="cuda")
    sizes = torch.full((world,), -1, dtype=torch.int64, device="cuda")
    for r in range(world):
        k = launches(lib.density_b200_cheetah_decode_shard_phase3, hs[r], sizes[r:r + 1].data_ptr(), seam[r].data_ptr(), st)
        assert k == (3 if ins[r].numel() else 1)        # verdict of the rounds, tail, seam words; an empty piece: its seam words
    torch.cuda.synchronize()
    for r in range(world):
        assert bool((outs[r][caps[r]:] == CANARY).all()), f"piece {r} written past cap"
        lib.density_b200_cheetah_decode_shard_destroy(hs[r])
    flags, total, _ = S.seam_verdict(seam)
    res = [outs[r][:max(int(sizes[r].item()), 0)].cpu().numpy() for r in range(world)]
    return flags, total, res, transfers.cpu().numpy(), seam.cpu().numpy()


def trace_of(data):
    enc = oracle.encode(ALG, data)
    return enc, P.trace(ALG, enc, data.size)


def slices(enc, tr, cuts):
    """the oracle's stream cut at the stream offsets of the shard cuts (byte offsets into the input, multiples of 128)"""
    offs = [int(tr.off[c // BS]) if c // BS < len(tr.off) else enc.size for c in cuts[:-1]] + [enc.size]
    return [enc[a:b] for a, b in zip(offs[:-1], offs[1:])]


def check_pieces(torch, lib, data, cuts, pieces, tr):
    """pieces decode to the shards at `cuts` with verdict 0, and the composed transfers are the traced automaton at every cut"""
    from density_b200 import sharded as S
    shards = [data[a:b] for a, b in zip(cuts[:-1], cuts[1:])]
    flags, total, outs, T, words = decode_prot_pieces(torch, lib, pieces, [max(s.size, 4) for s in shards])
    assert flags == 0 and total == data.size, (cuts, words)
    for r, s in enumerate(shards):
        assert outs[r].size == s.size and (outs[r] == s).all(), (cuts, r)
    for r in range(1, len(cuts) - 1):
        if cuts[r] == data.size:
            continue
        b = cuts[r] // BS
        want = S.decode_prot_candidate(tr.state[b], tr.counter[b] % 16)
        assert S.compose_decode_prot_transfers(T, r) == want, (cuts, r)
    return outs


def check_data(torch, lib, data, cuts, encoder=False):
    """the slices of the oracle's stream, and with encoder=True the pieces of the protected sharded Cheetah encoder, decode to the shards"""
    enc, tr = trace_of(data)
    check_pieces(torch, lib, data, cuts, slices(enc, tr, cuts), tr)
    if encoder:
        from test_gpu_sharded_cl_protected_encode import encode_shards
        pieces, (eflags, _, _), _ = encode_shards(torch, lib, ALG, data, cuts)
        assert eflags == 0
        check_pieces(torch, lib, data, cuts, pieces, tr)


def text(n, first_page=0):
    from density_b200 import synth
    return synth.synth_text(n, first_page=first_page).numpy()


def cuts_at(n, *units):
    return [0] + [u * 256 for u in units] + [n]


def test_noise_mixed_and_text(torch_cuda, lib):
    from density_b200 import synth
    for data in (payload("random", MIB + 77, 1), synth.synth_mixed(2 * MIB).numpy(), text(MIB + 3, first_page=3)):
        n = data.size
        check_data(torch_cuda, lib, data, cuts_at(n, 1111, 2003, 3001), encoder=True)
        check_data(torch_cuda, lib, data, cuts_at(n, *range(397, n // 256, n // 256 // 8)))


def test_noise_bursts_at_and_across_cuts(torch_cuda, lib):
    data = text(2 * MIB, first_page=2)
    rnd = payload("random", 64 * 1024, 7)
    cuts_b = [1000, 2501, 4097, 6000]
    for i, b in enumerate(cuts_b):          # a burst ending at the cut, one straddling it, one starting at it, one across
        lo = [b * 256 - 2048, b * 256 - 1024, b * 256, b * 256 - 512][i]
        ln = [2048, 2048, 4096, 768][i]
        data[lo:lo + ln] = rnd[i * 8192:i * 8192 + ln]
    check_data(torch_cuda, lib, data, cuts_at(data.size, *cuts_b), encoder=True)


def test_ragged_pieces_empty_pieces_and_short_tails(torch_cuda, lib):
    from density_b200 import synth
    mixed = synth.synth_mixed(MIB).numpy()
    rng = np.random.default_rng(5)
    for world in range(2, 10):
        tail = int(rng.integers(1, 200))
        d = np.concatenate([mixed[:(mixed.size // 256 - 1) * 256], payload("random", tail, world)])
        body = d.size // 256
        inner = sorted(int(v) for v in rng.choice(np.arange(1, body), world - 2, replace=False))
        check_data(torch_cuda, lib, d, [0] + [256 * u for u in inner] + [256 * body, d.size])
    d = mixed[:200 * 1024 + 3]
    n, nb = d.size, d.size // 256
    for cuts in ([0, 0, 0, 300 * 256, n],                      # an empty first piece (and a second): the stream start in piece 2
                 [0, 100 * 256, 100 * 256, 100 * 256, n],       # empty middle pieces
                 [0, 256, 512, 768, 1024, nb * 256, n]):        # 256-byte shards, and a last piece shorter than one block
        check_data(torch_cuda, lib, d, cuts, encoder=True)


def test_every_seam_case_is_accepted(torch_cuda, lib):
    from test_gpu_protection import _shard_cases
    n = 0
    for end, nxt, cut, bld in _shard_cases(ALG):
        data, _ = bld.realize()
        check_data(torch_cuda, lib, data, [0, cut, data.size])
        n += 1
    assert n >= 20


def test_copy_decisions_feed_each_other_across_shards(torch_cuda, lib):
    from test_gpu_sharded_cl_protected_encode import _feedback_input
    data = _feedback_input()
    check_data(torch_cuda, lib, data, cuts_at(data.size, 137, 300, 620, 900), encoder=True)


def _enc_and_cuts(data, shard_cuts):
    enc, tr = trace_of(data)
    return enc, [int(tr.off[c // BS]) if c < data.size else enc.size for c in shard_cuts]


def test_the_quiet_paths_refusals_are_accepted(torch_cuda, lib):
    """the four cases test_gpu_sharded_cheetah_decode.py::test_refusals sees refused by the quiet path decode here"""
    torch = torch_cuda
    t = text(2 * MIB, first_page=5)
    noise = splitmix_bytes(MIB, 12)
    cases = []
    d = np.concatenate([t[:MIB], noise[:256 * 1024], t[MIB:]])          # copy mode in piece 1
    cases.append((d, [0, MIB - 64 * 1024, d.size]))
    d = t.copy()                                                          # an incompressible block on each side of the cut
    d[MIB - 128:MIB + 128] = noise[:256]
    cases.append((d, [0, MIB, d.size]))
    d = t.copy()                                                          # piece 0 ends with a copy penalty pending
    d[MIB - 256:MIB] = noise[:256]
    cases.append((d, [0, MIB, d.size]))
    d = np.concatenate([t[:MIB], noise[:64 * 1024], t[MIB:]])            # piece 0 ends inside a copy run
    cases.append((d, [0, MIB + 64 * 1024, d.size]))
    for d, cuts in cases:
        enc, pc = _enc_and_cuts(d, cuts)
        pieces = [enc[a:b] for a, b in zip(pc[:-1], pc[1:])]
        flags, total, outs, _, _ = decode_prot_pieces(torch, lib, pieces, [cuts[1], d.size - cuts[1]])
        assert flags == 0 and total == d.size and (np.concatenate(outs) == d).all(), cuts


def test_a_moved_cut_a_short_cap_and_a_small_round_budget_are_refused(torch_cuda, lib):
    torch = torch_cuda
    data = text(2 * MIB)
    data[MIB - 4096:MIB + 4096] = payload("random", 8192, 3)
    enc, tr = trace_of(data)
    assert tr.copied.any()
    cuts = [0, MIB - 3 * BS, MIB + 5 * BS, data.size]
    offs = [int(tr.off[c // BS]) for c in cuts[:-1]] + [enc.size]
    caps = [cuts[1] - cuts[0], cuts[2] - cuts[1], cuts[3] - cuts[2]]
    for delta in (2, -2):
        o = list(offs)
        o[1] += delta
        flags, _, _, _, _ = decode_prot_pieces(torch, lib, [enc[a:b] for a, b in zip(o[:-1], o[1:])], [c + 1024 for c in caps])
        assert flags != 0, delta
    pieces = [enc[a:b] for a, b in zip(offs[:-1], offs[1:])]
    flags, total, outs, _, _ = decode_prot_pieces(torch, lib, pieces, caps)
    assert flags == 0 and total == data.size and (np.concatenate(outs) == data).all()
    for r in range(3):
        short = list(caps)
        short[r] -= 128
        flags, _, _, _, words = decode_prot_pieces(torch, lib, pieces, short)
        assert flags != 0 and words[r][2] == 1, r
    lib.density_b200_test_set_decode_rounds(1)
    try:
        flags, _, _, _, words = decode_prot_pieces(torch, lib, pieces, caps)
        assert flags != 0
    finally:
        lib.density_b200_test_set_decode_rounds(40)


def _decode_device(torch, data_enc, cap):
    import density_b200
    d_in = torch.from_numpy(data_enc.copy()).cuda()
    d_out = torch.zeros(max(cap, 4), dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    density_b200.decode_device(ALG, d_in, d_in.numel(), d_out, d_sz)
    torch.cuda.synchronize()
    return d_out[:int(d_sz.item())].cpu().numpy()


def test_damaged_pieces_refuse_or_match_decode_device(torch_cuda, lib):
    torch = torch_cuda
    data = text(MIB + 77, first_page=4)
    data[MIB // 2:MIB // 2 + 32 * 1024] = payload("random", 32 * 1024, 4)
    cuts = [0, MIB // 2 + 16 * 1024, data.size]
    enc, pc = _enc_and_cuts(data, cuts)
    rng = np.random.default_rng(5)
    for trial in range(8):
        e = enc.copy()
        if trial < 4:
            k = int(rng.integers(pc[1] // 2, e.size))
            e[k] ^= np.uint8(1 << int(rng.integers(0, 8)))
            p = list(pc)
        else:
            c = int(rng.integers(1, 300))
            e = np.concatenate([enc[:pc[1] - c], enc[pc[1]:]]) if trial < 6 else enc[:-c]
            p = [0, pc[1] - c, e.size] if trial < 6 else [0, pc[1], e.size]
        flags, _, got, _, _ = decode_prot_pieces(torch, lib, [e[a:b] for a, b in zip(p[:-1], p[1:])], [16 * e.size + 256] * 2)
        if flags == 0:
            want = _decode_device(torch, e, 16 * e.size + 256)
            cat = np.concatenate(got)
            assert cat.size == want.size and (cat == want).all(), trial


def test_argument_and_phase_order_errors_enqueue_nothing(torch_cuda, lib):
    torch = torch_cuda
    st = _stream(torch)
    h = lib.density_b200_cheetah_decode_shard_create()
    d_in = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(65536, dtype=torch.uint8, device="cuda")
    tr = torch.zeros(2 * 3200, dtype=torch.int32, device="cuda")
    t = torch.zeros(3 * 65536, dtype=torch.int32, device="cuda")
    w = torch.zeros(8, dtype=torch.int32, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    xfer = lib.density_b200_cheetah_decode_shard_prot_transfer
    ph1 = lib.density_b200_cheetah_decode_shard_prot_phase1
    before = lib.density_b200_kernel_launches()
    assert ph1(h, tr.data_ptr(), 2, 1, t.data_ptr(), st) == EARG                                              # no transfer
    assert xfer(h, d_in.data_ptr() + 1, 1024, d_out.data_ptr(), 65536, 1, 0, tr.data_ptr(), st) == EARG         # d_in misaligned
    assert xfer(h, d_in.data_ptr(), 1024, d_out.data_ptr() + 2, 65536, 1, 0, tr.data_ptr(), st) == EARG         # d_out misaligned
    assert xfer(h, d_in.data_ptr(), 1024, d_out.data_ptr(), 65536, 1, 0, tr.data_ptr() + 2, st) == EARG         # transfer misaligned
    assert xfer(h, d_in.data_ptr(), 1024, d_out.data_ptr(), 65536, 1, 0, None, st) == EARG
    assert xfer(h, None, 1024, d_out.data_ptr(), 65536, 1, 0, tr.data_ptr(), st) == EARG
    assert lib.density_b200_kernel_launches() == before
    assert xfer(h, d_in.data_ptr(), 1024, d_out.data_ptr(), 65536, 0, 0, tr[3200:].data_ptr(), st) == 0
    before = lib.density_b200_kernel_launches()
    assert lib.density_b200_cheetah_decode_shard_phase2(h, None, st) == EARG                                     # prot_phase1 not done
    assert ph1(h, tr.data_ptr(), 2, 2, t.data_ptr(), st) == EARG                                                 # rank >= world
    assert ph1(h, tr.data_ptr(), 0, 0, t.data_ptr(), st) == EARG
    assert ph1(h, tr.data_ptr(), 2, -1, t.data_ptr(), st) == EARG
    assert ph1(h, None, 2, 1, t.data_ptr(), st) == EARG                                                          # rank > 0 needs them
    assert ph1(h, tr.data_ptr() + 2, 2, 1, t.data_ptr(), st) == EARG
    assert ph1(h, tr.data_ptr(), 2, 1, t.data_ptr() + 2, st) == EARG
    assert lib.density_b200_kernel_launches() == before
    # a quiet phase 1 in between closes the protected sequence
    assert lib.density_b200_cheetah_decode_shard_phase1(h, d_in.data_ptr(), 1024, d_out.data_ptr(), 65536, 1, 1, None, st) == 0
    before = lib.density_b200_kernel_launches()
    assert ph1(h, tr.data_ptr(), 2, 1, t.data_ptr(), st) == EARG
    assert lib.density_b200_kernel_launches() == before
    # the right order works, once
    assert xfer(h, d_in.data_ptr(), 1024, d_out.data_ptr(), 65536, 0, 1, tr[3200:].data_ptr(), st) == 0
    assert ph1(h, tr.data_ptr(), 2, 1, None, st) == 0
    assert ph1(h, tr.data_ptr(), 2, 1, None, st) == EARG                                                         # one phase 1 per transfer
    assert lib.density_b200_cheetah_decode_shard_phase3(h, sz.data_ptr(), w.data_ptr(), st) == EARG             # phase 2 not done
    assert lib.density_b200_cheetah_decode_shard_phase2(h, None, st) == 0
    assert lib.density_b200_cheetah_decode_shard_round_walk(h, None, w.data_ptr(), st) == 0
    assert lib.density_b200_cheetah_decode_shard_round_fold(h, None, w.data_ptr(), 2, 1, st) == 0
    assert lib.density_b200_cheetah_decode_shard_phase3(h, sz.data_ptr(), w.data_ptr(), st) == 0
    torch.cuda.synchronize()
    lib.density_b200_cheetah_decode_shard_destroy(h)
    from density_b200 import sharded
    dec = sharded.ShardedDecoder(torch.device("cuda"))
    fl = torch.zeros(1, dtype=torch.int32, device="cuda")
    before = lib.density_b200_kernel_launches()
    fn = lib.density_b200_decode_sharded_cheetah_protected
    assert fn(dec._h, d_in.data_ptr() + 1, 1024, d_out.data_ptr(), 65536, sz.data_ptr(), fl.data_ptr(), None, st) == EARG
    assert fn(dec._h, d_in.data_ptr(), 1024, d_out.data_ptr() + 2, 65536, sz.data_ptr(), fl.data_ptr(), None, st) == EARG
    assert fn(dec._h, d_in.data_ptr(), 1024, d_out.data_ptr(), 65536, None, fl.data_ptr(), None, st) == EARG
    assert lib.density_b200_kernel_launches() == before
    with pytest.raises(ValueError):
        dec.decode_protected(d_in, d_out, sz, fl, alg="lion")
    dec.close()


def test_driver_world_one_and_python_equal_decode_device(torch_cuda, lib):
    """density_b200_decode_sharded_cheetah_protected with one rank (no NCCL) and ShardedDecoder.decode_protected(alg="cheetah") equal
    decode_device; the driver enqueues two kernels more than density_b200_decode_sharded_cheetah (the transfer's head walk and the seed;
    the boundary kernels reuse the transfer's candidate rows)."""
    torch = torch_cuda
    from density_b200 import sharded, synth
    dec = sharded.ShardedDecoder(torch.device("cuda"))
    st = _stream(torch)
    for data in (text(5 * MIB + 1021), synth.synth_mixed(3 * MIB).numpy(), payload("random", MIB + 5, 6), np.zeros(MIB + 3, np.uint8),
                 text(77, 3)):
        enc = oracle.encode(ALG, data)
        want = _decode_device(torch, enc, data.size + 64)
        assert (want == data).all()
        d_in = torch.from_numpy(enc.copy()).cuda()
        d_out = torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_fl = torch.ones(1, dtype=torch.int32, device="cuda")
        dec.decode_protected(d_in, d_out, d_sz, d_fl, alg="cheetah")
        torch.cuda.synchronize()
        assert int(d_fl.item()) == 0 and int(d_sz.item()) == data.size == int(dec.d_total.item())
        assert (d_out[:data.size].cpu().numpy() == want).all()
        counts = []
        for fn in (lib.density_b200_decode_sharded_cheetah_protected, lib.density_b200_decode_sharded_cheetah):
            d_out.zero_()
            before = lib.density_b200_kernel_launches()
            assert fn(dec._h, d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), d_out.numel(), d_sz.data_ptr(), d_fl.data_ptr(), None, st) == 0
            counts.append(lib.density_b200_kernel_launches() - before)
            torch.cuda.synchronize()
            if fn is lib.density_b200_decode_sharded_cheetah_protected:
                assert int(d_fl.item()) == 0 and (d_out[:data.size].cpu().numpy() == want).all()
        assert counts[0] == counts[1] + 2, counts
    dec.close()


def _nccl_worker(rank, world, port, n_per_rank, q):
    import os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import density_b200
    from density_b200 import sharded, synth
    enc = sharded.ShardedEncoder(dev)
    d_in = synth.synth_mixed(n_per_rank, device=dev) if rank % 2 else synth.synth_text(n_per_rank, device=dev, first_page=rank)
    cap = density_b200.load().cheetah_safe_encode_buffer_size(n_per_rank)
    d_piece = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    enc.encode_protected(d_in, d_piece, d_sz, d_fl, alg="cheetah")
    torch.cuda.synchronize()
    fl_enc = int(d_fl.item())
    piece = d_piece[:int(d_sz.item())].clone()
    dec = sharded.ShardedDecoder(dev)
    d_out = torch.zeros(n_per_rank + 64, dtype=torch.uint8, device=dev)
    d_fl.fill_(1)
    dec.decode_protected(piece, d_out, d_sz, d_fl, alg="cheetah")
    torch.cuda.synchronize()
    ok = int(d_sz.item()) == n_per_rank and bool((d_out[:n_per_rank] == d_in).all().item())
    q.put((rank, fl_enc, int(d_fl.item()), ok, int(dec.d_total.item())))
    dist.barrier()
    enc.close(); dec.close()
    dist.destroy_process_group()


def test_decode_sharded_cheetah_protected_two_ranks_nccl(torch_cuda):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, n_per = 2, 8 * MIB
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, 29743, n_per, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r, *rest = q.get(timeout=600)
        got[r] = rest
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert all(got[r] == [0, 0, True, world * n_per] for r in range(world)), got
