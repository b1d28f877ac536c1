"""Sharded Lion decode through the phase API on one device (needs an H100: pytest -m gpu).

W pieces run density_b200_lion_decode_shard_phase1, phase 2, the walk and phase 3, the chunk-map exchange replaced by stacking the
transfers and folding them with the library's fold, and the relay of the walk's state by handing one device buffer from piece to piece
in rank order. Every piece of the sharded Lion encoder, and every slice of one lion_encode stream at the same prefix sums, decodes to its
shard byte for byte with verdict 0; the quiet path refuses what it cannot decode; damaged pieces refuse or decode as decode_device does."""
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
ALG = "lion"
BS = P.BS[ALG]
STATE_WORDS = 5 * 65536 + 8          # DENSITY_B200_LION_STATE_WORDS


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


def decode_lion_pieces(torch, lib, pieces, caps, prot=False):
    """Every phase of every piece on one device, the walk's state relayed through one buffer. Returns (flags, total, outs, seam words
    [W, 8], per-piece walk counts [W, 4], transfers [W, 3200] or None). Checks that nothing is written past cap and pins the launches of
    every phase."""
    from density_b200 import sharded as S
    world, st = len(pieces), _stream(torch)
    wc = lib.density_b200_cheetah_cmap_words()
    hs = [lib.density_b200_lion_decode_shard_create() for _ in range(world)]
    ins = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in pieces]
    outs = [torch.full((caps[r] + 64,), CANARY, dtype=torch.uint8, device="cuda") for r in range(world)]
    tc = torch.zeros((world, wc), dtype=torch.int32, device="cuda")
    transfers = torch.full((world, S.DECODE_PROT_TRANSFER_WORDS), -1, dtype=torch.int32, device="cuda") if prot else None

    def launches(fn, *args):
        before = lib.density_b200_kernel_launches()
        rc = fn(*args)
        assert rc == 0, lib.density_b200_last_error()
        return lib.density_b200_kernel_launches() - before

    first = next((r for r in range(world) if pieces[r].size), 0)      # the piece that holds the stream start
    if prot:
        for r in range(world):
            n = ins[r].numel()
            k = launches(lib.density_b200_lion_decode_shard_prot_transfer, hs[r], _ptr(ins[r]), n, outs[r].data_ptr(), caps[r],
                         int(r == first), int(r == world - 1), transfers[r].data_ptr(), st)
            assert k == (3 if n else 1)                  # candidate rows, group rows, head walk
    for r in range(world):
        n, last = ins[r].numel(), r == world - 1
        cm = None if last else tc[r].data_ptr()
        if prot:
            k = launches(lib.density_b200_lion_decode_shard_prot_phase1, hs[r], transfers.data_ptr(), world, r, cm, st)
            assert k == 1 + (7 + 1 + 2 if n else 0) + (0 if last else 1), (r, k)   # seed, boundaries on the rows, end, unpack + walk, export
        else:
            k = launches(lib.density_b200_lion_decode_shard_phase1, hs[r], _ptr(ins[r]), n, outs[r].data_ptr(), caps[r], int(r == first),
                         int(last), cm, st)
            assert k == (9 + 1 + 2 if n else 0) + (0 if last else 1), (r, k)
    for r in range(world):
        carry = S.fold_cheetah_cmap(tc, r) if r > 0 else None
        k = launches(lib.density_b200_lion_decode_shard_phase2, hs[r], carry.data_ptr() if carry is not None else None, st)
        assert k == (2 if ins[r].numel() else 0)
    state = torch.full((STATE_WORDS,), -1, dtype=torch.int32, device="cuda")
    assert lib.density_b200_lion_state_init(state.data_ptr(), st) == 0
    for r in range(world):
        k = launches(lib.density_b200_lion_decode_shard_walk, hs[r], state.data_ptr(), st)
        assert k == (1 if ins[r].numel() else 0)
    seam = torch.zeros((world, 8), dtype=torch.int32, device="cuda")
    sizes = torch.full((world,), -1, dtype=torch.int64, device="cuda")
    for r in range(world):
        k = launches(lib.density_b200_lion_decode_shard_phase3, hs[r], sizes[r:r + 1].data_ptr(), seam[r].data_ptr(), st)
        assert k == (3 if ins[r].numel() else (1 if prot else 0))    # verdict of the walk, tail, seam words
    torch.cuda.synchronize()
    counts = np.zeros((world, 4), np.uint64)
    for r in range(world):
        assert bool((outs[r][caps[r]:] == CANARY).all()), f"piece {r} written past cap"
        c = (ctypes.c_uint64 * 4)()
        assert lib.density_b200_lion_decode_shard_stats(hs[r], c) == 0
        counts[r] = list(c)
        lib.density_b200_lion_decode_shard_destroy(hs[r])
    flags, total, _ = S.seam_verdict(seam)
    res = [outs[r][:max(int(sizes[r].item()), 0)].cpu().numpy() for r in range(world)]
    return flags, total, res, seam.cpu().numpy(), counts, transfers.cpu().numpy() if prot else None


def trace_of(data):
    enc = oracle.encode(ALG, data)
    return enc, P.trace(ALG, enc, data.size)


def slices(enc, tr, cuts):
    """the oracle's stream cut at the stream offsets of the shard cuts (byte offsets into the input, multiples of 64)"""
    offs = [int(tr.off[c // BS]) if c // BS < len(tr.off) else enc.size for c in cuts[:-1]] + [enc.size]
    return [enc[a:b] for a, b in zip(offs[:-1], offs[1:])]


def single_counts(torch, lib, enc, n):
    """decode_device of the whole stream: (output, its walk counts)"""
    import density_b200
    d_in = torch.from_numpy(enc.copy()).cuda()
    d_out = torch.zeros(max(n, 4) + 64, dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    density_b200.decode_device(ALG, d_in, d_in.numel(), d_out, d_sz)
    torch.cuda.synchronize()
    c = (ctypes.c_uint64 * 4)()
    rc = lib.density_b200_lion_decode_stats(c)
    return d_out[:int(d_sz.item())].cpu().numpy(), (list(c) if rc == 0 else None)


def check_pieces(torch, lib, data, cuts, pieces, prot=False, want_counts=None):
    shards = [data[a:b] for a, b in zip(cuts[:-1], cuts[1:])]
    flags, total, outs, words, counts, _ = decode_lion_pieces(torch, lib, pieces, [max(s.size, 4) for s in shards], prot)
    assert flags == 0 and total == data.size, (cuts, words)
    for r, s in enumerate(shards):
        assert outs[r].size == s.size and (outs[r] == s).all(), (cuts, r)
    # quads and predicted quads walked add up to the single call's, unless the single call's tail (the blocks in the stream's last 70
    # bytes) starts in front of the last piece: a non-final piece walks all of its blocks
    if want_counts is not None and pieces[-1].size >= 70:
        assert int(counts[:, 0].sum()) == want_counts[0] and int(counts[:, 1].sum()) == want_counts[1], (counts, want_counts)
    return counts


def check_data(torch, lib, data, cuts, encoder=True, prot=False):
    """the slices of the oracle's stream, and with encoder=True the pieces of the sharded Lion encoder (the protected one with prot),
    decode to the shards; the walk counts of the pieces add up to decode_device's"""
    enc, tr = trace_of(data)
    got, want_counts = single_counts(torch, lib, enc, data.size)
    assert (got == data).all()
    check_pieces(torch, lib, data, cuts, slices(enc, tr, cuts), prot, want_counts)
    if encoder:
        if prot:
            from test_gpu_sharded_cl_protected_encode import encode_shards
            pieces, (eflags, _, _), _ = encode_shards(torch, lib, ALG, data, cuts)
        else:
            from test_gpu_sharded_cl_encode import encode_shards
            pieces, (eflags, _, _), _ = encode_shards(torch, lib, ALG, data, cuts)
        assert eflags == 0
        check_pieces(torch, lib, data, cuts, pieces, prot, want_counts)


def text(n, first_page=0):
    from density_b200 import synth
    return synth.synth_text(n, first_page=first_page).numpy()


def even_cuts(n, world):
    step = n // world // 256 * 256
    return [0] + [step * r for r in range(1, world)] + [n]


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_pieces_decode_to_their_shards_text(torch_cuda, lib, world):
    data = text(2 * MIB + 333, first_page=world)
    check_data(torch_cuda, lib, data, even_cuts(data.size, world))


@pytest.mark.parametrize("world", [2, 4, 7])
def test_pieces_decode_to_their_shards_dickens_and_zeros(torch_cuda, lib, dickens200k, world):
    """quiet data (mixed data and noise have copy mode after the first piece: the protected tests decode them)"""
    for data in (dickens200k, np.zeros(MIB + 5, np.uint8)):
        check_data(torch_cuda, lib, data, even_cuts(data.size, world))


def test_noise_is_quiet_after_the_start(torch_cuda, lib):
    """noise: incompressible blocks throughout, so copy mode everywhere; one piece decodes, and the protected test file covers more"""
    data = payload("random", 300 * 1024 + 7, 3)
    check_data(torch_cuda, lib, data, [0, data.size])


def test_empty_pieces_start_behind_them_and_a_tiny_last_piece(torch_cuda, lib):
    d = text(600 * 1024 + 3, first_page=2)
    n, nb = d.size, d.size // 256
    for cuts in ([0, 0, 0, 300 * 256, n],                          # the stream start on rank 2, behind two empty pieces
                 [0, 100 * 256, 100 * 256, 100 * 256, n],           # empty middle pieces
                 [0, 100 * 256, 101 * 256, 102 * 256, nb * 256, n], # 256-byte shards (behind the stream start's copy run), a tiny last piece
                 [0, nb * 256, nb * 256, n]):                       # an empty piece in front of the tail
        check_data(torch_cuda, lib, d, cuts, encoder=cuts[1] > 0)   # the sharded encoder puts the stream start on rank 0


def _enc_and_cuts(data, shard_cuts):
    enc, tr = trace_of(data)
    return enc, [int(tr.off[c // BS]) if c < data.size else enc.size for c in shard_cuts]


def test_refusals(torch_cuda, lib):
    """every refusal of the quiet path fires, on the seam word of the piece that causes it"""
    torch = torch_cuda
    t = text(2 * MIB, first_page=5)
    noise = splitmix_bytes(MIB, 12)

    def run(d, cuts, enc=None, pc=None):
        if enc is None:
            enc, pc = _enc_and_cuts(d, cuts)
        caps = [max(b - a, 4) + 1024 for a, b in zip(cuts[:-1], cuts[1:])]
        return decode_lion_pieces(torch, lib, [enc[a:b] for a, b in zip(pc[:-1], pc[1:])], caps)
    # copy mode in piece 1
    d = np.concatenate([t[:MIB], noise[:256 * 1024], t[MIB:]])
    flags, _, _, words, _, _ = run(d, [0, MIB - 64 * 1024, d.size])
    assert flags != 0 and words[1][2] == 1 and words[0][2] == 0
    # an incompressible block on each side of a seam
    d = t.copy()
    d[MIB - 64:MIB + 64] = noise[:128]
    flags, _, _, words, _, _ = run(d, [0, MIB, d.size])
    assert flags != 0 and words[0][1] == 1 and words[1][0] == 1 and words[0][2] == 0
    # piece 0 ends with a copy penalty pending
    d = t.copy()
    d[MIB - 128:MIB] = noise[:128]
    flags, _, _, words, _, _ = run(d, [0, MIB, d.size])
    assert flags != 0 and words[0][2] == 1
    # piece 0 ends inside a copy run
    d = np.concatenate([t[:MIB], noise[:64 * 1024], t[MIB:]])
    flags, _, _, words, _, _ = run(d, [0, MIB + 64 * 1024, d.size])
    assert flags != 0 and words[0][2] == 1
    # a non-final piece whose blocks do not end at its last byte, and a short cap
    d = t[:MIB + 99]
    enc, pc = _enc_and_cuts(d, [0, MIB // 2, d.size])
    for delta in (2, -2):
        p = [0, pc[1] + delta, enc.size]
        flags, _, _, words, _, _ = run(d, [0, MIB // 2, d.size], enc, p)
        assert flags != 0, delta
    flags, _, _, words, _, _ = decode_lion_pieces(torch, lib, [enc[:pc[1]], enc[pc[1]:]], [MIB // 2 - 64, d.size - MIB // 2])
    assert flags != 0 and words[0][2] == 1


def test_damaged_pieces_refuse_or_match_decode_device(torch_cuda, lib):
    torch = torch_cuda
    data = text(MIB + 77, first_page=4)
    cuts = [0, MIB // 2, data.size]
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
        flags, _, got, _, _, _ = decode_lion_pieces(torch, lib, [e[a:b] for a, b in zip(p[:-1], p[1:])], [16 * e.size + 256] * 2)
        if flags == 0:
            want, _ = single_counts(torch, lib, e, 16 * e.size + 256)
            cat = np.concatenate(got)
            assert cat.size == want.size and (cat == want).all(), trial


def test_argument_and_phase_order_errors_enqueue_nothing(torch_cuda, lib):
    torch = torch_cuda
    st = _stream(torch)
    h = lib.density_b200_lion_decode_shard_create()
    enc = oracle.encode(ALG, text(4000))
    d_in = torch.from_numpy(np.concatenate([enc, np.zeros(8, np.uint8)])).cuda()
    n = enc.size
    d_out = torch.zeros(65536, dtype=torch.uint8, device="cuda")
    t = torch.zeros(3 * 65536, dtype=torch.int32, device="cuda")
    state = torch.zeros(STATE_WORDS + 1, dtype=torch.int32, device="cuda")
    w = torch.zeros(8, dtype=torch.int32, device="cuda")
    sz = torch.zeros(2, dtype=torch.int64, device="cuda")
    ph1, ph2 = lib.density_b200_lion_decode_shard_phase1, lib.density_b200_lion_decode_shard_phase2
    walk, ph3 = lib.density_b200_lion_decode_shard_walk, lib.density_b200_lion_decode_shard_phase3
    out4 = (ctypes.c_uint64 * 4)()
    before = lib.density_b200_kernel_launches()
    assert ph2(h, None, st) == EARG and walk(h, state.data_ptr(), st) == EARG                        # phase 1 not done
    assert ph3(h, sz.data_ptr(), w.data_ptr(), st) == EARG and lib.density_b200_lion_decode_shard_stats(h, out4) == EARG
    assert ph1(h, d_in.data_ptr() + 1, n, d_out.data_ptr(), 65536, 1, 1, None, st) == EARG              # d_in misaligned
    assert ph1(h, d_in.data_ptr(), n, d_out.data_ptr() + 2, 65536, 1, 1, None, st) == EARG              # d_out misaligned
    assert ph1(h, d_in.data_ptr(), n, d_out.data_ptr(), 65536, 1, 0, t.data_ptr() + 2, st) == EARG      # table misaligned
    assert ph1(h, None, n, d_out.data_ptr(), 65536, 1, 1, None, st) == EARG
    assert ph1(h, d_in.data_ptr(), n, None, 65536, 1, 1, None, st) == EARG
    assert lib.density_b200_lion_state_init(None, st) == EARG and lib.density_b200_lion_state_init(state.data_ptr() + 2, st) == EARG
    assert lib.density_b200_lion_decode_shard_prot_phase1(h, None, 1, 0, None, st) == EARG             # no transfer
    assert lib.density_b200_kernel_launches() == before
    assert ph1(h, d_in.data_ptr(), n, d_out.data_ptr(), 65536, 1, 1, None, st) == 0
    before = lib.density_b200_kernel_launches()
    assert walk(h, state.data_ptr(), st) == EARG and ph3(h, sz.data_ptr(), w.data_ptr(), st) == EARG     # phase 2 not done
    assert ph2(h, t.data_ptr() + 2, st) == EARG
    assert lib.density_b200_kernel_launches() == before
    assert ph2(h, None, st) == 0
    before = lib.density_b200_kernel_launches()
    assert ph2(h, None, st) == EARG                                                                     # one phase 2 per phase 1
    assert ph3(h, sz.data_ptr(), w.data_ptr(), st) == EARG                                              # the walk not done
    assert walk(h, None, st) == EARG and walk(h, state.data_ptr() + 2, st) == EARG
    assert lib.density_b200_kernel_launches() == before
    assert lib.density_b200_lion_state_init(state.data_ptr(), st) == 0
    assert walk(h, state.data_ptr(), st) == 0
    before = lib.density_b200_kernel_launches()
    assert walk(h, state.data_ptr(), st) == EARG
    assert ph3(h, None, w.data_ptr(), st) == EARG and ph3(h, sz.data_ptr(), None, st) == EARG
    assert ph3(h, sz.data_ptr() + 4, w.data_ptr(), st) == EARG and ph3(h, sz.data_ptr(), w.data_ptr() + 2, st) == EARG
    assert lib.density_b200_kernel_launches() == before
    assert ph3(h, sz.data_ptr(), w.data_ptr(), st) == 0
    assert lib.density_b200_lion_decode_shard_stats(h, out4) == 0
    torch.cuda.synchronize()
    assert int(sz[0].item()) == 4000 and list(out4)[0] > 0
    before = lib.density_b200_kernel_launches()
    assert ph3(h, sz.data_ptr(), w.data_ptr(), st) == EARG                                              # one phase 3 per phase 1
    assert lib.density_b200_kernel_launches() == before
    lib.density_b200_lion_decode_shard_destroy(h)
    from density_b200 import sharded
    dec = sharded.ShardedLionDecoder(torch.device("cuda"))
    fl = torch.zeros(1, dtype=torch.int32, device="cuda")
    before = lib.density_b200_kernel_launches()
    for fn in (lib.density_b200_decode_sharded_lion, lib.density_b200_decode_sharded_lion_protected):
        assert fn(dec._h, d_in.data_ptr() + 1, n, d_out.data_ptr(), 65536, sz.data_ptr(), fl.data_ptr(), None, st) == EARG
        assert fn(dec._h, d_in.data_ptr(), n, d_out.data_ptr() + 2, 65536, sz.data_ptr(), fl.data_ptr(), None, st) == EARG
        assert fn(dec._h, d_in.data_ptr(), n, d_out.data_ptr(), 65536, None, fl.data_ptr(), None, st) == EARG
        assert fn(dec._h, d_in.data_ptr(), n, d_out.data_ptr(), 65536, sz.data_ptr() + 4, fl.data_ptr(), None, st) == EARG
    assert lib.density_b200_kernel_launches() == before
    dec.close()
    # ShardedDecoder keeps refusing Lion
    dec = sharded.ShardedDecoder(torch.device("cuda"))
    for fn in (dec.decode, dec.decode_protected):
        with pytest.raises(ValueError, match="ShardedLionDecoder"):
            fn(d_in, d_out, sz[:1], fl, alg="lion")
    dec.close()


def test_decode_device_keeps_its_lion_launches_and_stats(torch_cuda, lib, dickens200k):
    """decode_device: 9 boundary kernels, unpack, chunk-map walk, fold, resolve, the walk, the verdict, the tail and the in-order kernel
    behind it; the stats are the walk's counts"""
    import density_b200
    torch = torch_cuda
    data = dickens200k
    enc = oracle.encode(ALG, data)
    d_in = torch.from_numpy(enc).cuda()
    d_out = torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    before = lib.density_b200_kernel_launches()
    density_b200.decode_device(ALG, d_in, enc.size, d_out, d_sz)
    torch.cuda.synchronize()
    assert lib.density_b200_kernel_launches() - before == 17
    assert int(d_sz.item()) == data.size and (d_out[:data.size].cpu().numpy() == data).all()
    c = (ctypes.c_uint64 * 4)()
    assert lib.density_b200_lion_decode_stats(c) == 0
    q = list(c)
    assert q[0] > 0 and q[3] > 0
    # the one-piece phase run walks the same quads
    counts = check_pieces(torch, lib, data, [0, data.size], [enc])
    assert list(counts[0]) == q


def test_driver_world_one_and_python_equal_decode_device(torch_cuda, lib):
    """density_b200_decode_sharded_lion(_protected) with one rank (no NCCL) and ShardedLionDecoder equal decode_device; the protected
    driver enqueues two kernels more (the transfer's head walk and the seed)"""
    torch = torch_cuda
    from density_b200 import sharded, synth
    dec = sharded.ShardedLionDecoder(torch.device("cuda"))
    st = _stream(torch)
    for data in (text(3 * MIB + 1021), synth.synth_mixed(MIB).numpy(), payload("random", MIB + 5, 6), np.zeros(MIB + 3, np.uint8),
                 text(77, 3)):
        enc = oracle.encode(ALG, data)
        want, _ = single_counts(torch, lib, enc, data.size)
        assert (want == data).all()
        d_in = torch.from_numpy(enc.copy()).cuda()
        d_out = torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_fl = torch.ones(1, dtype=torch.int32, device="cuda")
        for py in (dec.decode, dec.decode_protected):
            d_out.zero_(); d_fl.fill_(1)
            py(d_in, d_out, d_sz, d_fl)
            torch.cuda.synchronize()
            assert int(d_fl.item()) == 0 and int(d_sz.item()) == data.size == int(dec.d_total.item())
            assert (d_out[:data.size].cpu().numpy() == want).all()
        counts = []
        for fn in (lib.density_b200_decode_sharded_lion_protected, lib.density_b200_decode_sharded_lion):
            before = lib.density_b200_kernel_launches()
            assert fn(dec._h, d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), d_out.numel(), d_sz.data_ptr(), d_fl.data_ptr(), None, st) == 0
            counts.append(lib.density_b200_kernel_launches() - before)
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
    cap = density_b200.load().lion_safe_encode_buffer_size(n_per_rank)
    d_piece = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    enc.encode_protected(d_in, d_piece, d_sz, d_fl, alg="lion")
    torch.cuda.synchronize()
    fl_enc = int(d_fl.item())
    piece = d_piece[:int(d_sz.item())].clone()
    dec = sharded.ShardedLionDecoder(dev)
    d_out = torch.zeros(n_per_rank + 64, dtype=torch.uint8, device=dev)
    d_fl.fill_(1)
    dec.decode_protected(piece, d_out, d_sz, d_fl)
    torch.cuda.synchronize()
    ok = int(d_sz.item()) == n_per_rank and bool((d_out[:n_per_rank] == d_in).all().item())
    q.put((rank, fl_enc, int(d_fl.item()), ok, int(dec.d_total.item())))
    dist.barrier()
    enc.close(); dec.close()
    dist.destroy_process_group()


def test_decode_sharded_lion_protected_two_ranks_nccl(torch_cuda):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, n_per = 2, 4 * MIB
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, 29751, n_per, q)) for r in range(world)]
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
