"""Sharded Chameleon decode of streams with copy-mode blocks, through the phase API on one device (needs an H100: pytest -m gpu).

W pieces run density_b200_decode_shard_prot_transfer / _phase1 / _phase2 on one device, the exchanges replaced by stacking the
transfers, tables and seam words and folding the tables with sharded.fold_tables. Whatever the data -- noise, synth_mixed, text with
noise bursts at the cuts, automaton states and pending penalties on the cuts, copy decisions that feed each other -- every piece of
the protected sharded encoder, and every slice of one chameleon_encode stream at the same prefix sums, decodes to its shard byte for
byte with verdict 0, and the composed transfers are the in-order automaton of the stream at every cut."""
import ctypes

import numpy as np
import pytest

import oracle
import protection as P
from conftest import payload

pytestmark = pytest.mark.gpu

MIB = 1 << 20
CANARY = 0xA5


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


def decode_prot_pieces(torch, lib, pieces, caps):
    """Every phase of every piece on one device. Returns (flags, total, outs, transfers [W, 3200] as numpy)."""
    from density_b200 import sharded as S
    world = len(pieces)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    decs = [S.ShardedChameleonDecoder() for _ in range(world)]
    ins = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in pieces]
    ptr = [t.data_ptr() if t.numel() else None for t in ins]
    transfers = torch.full((world, S.DECODE_PROT_TRANSFER_WORDS), -1, dtype=torch.int32, device="cuda")
    for r in range(world):
        rc = lib.density_b200_decode_shard_prot_transfer(decs[r]._h, ptr[r], ins[r].numel(), caps[r], int(r == world - 1),
                                                         transfers[r].data_ptr(), st)
        assert rc == 0, lib.density_b200_last_error()
    tables = torch.empty((world, S.TABLE_ENTRIES), dtype=torch.int32, device="cuda")
    for r in range(world):
        rc = lib.density_b200_decode_shard_prot_phase1(decs[r]._h, transfers.data_ptr(), world, r, tables[r].data_ptr(), st)
        assert rc == 0, lib.density_b200_last_error()
    seams = torch.zeros((world, S.SEAM_WORDS), dtype=torch.int32, device="cuda")
    outs, sizes = [], []
    for r in range(world):
        carry = S.fold_tables(tables, r).contiguous()
        d_out = torch.full((caps[r] + 64,), CANARY, dtype=torch.uint8, device="cuda")
        d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        rc = lib.density_b200_decode_shard_prot_phase2(decs[r]._h, carry.data_ptr(), d_out.data_ptr(), d_sz.data_ptr(), seams[r].data_ptr(), st)
        assert rc == 0, lib.density_b200_last_error()
        outs.append(d_out); sizes.append(d_sz)
    torch.cuda.synchronize()
    for r in range(world):
        assert bool((outs[r][caps[r]:] == CANARY).all()), f"piece {r} written past cap"
    flags, total, _ = S.seam_verdict(seams)
    res = [outs[r][:max(int(sizes[r].item()), 0)].cpu().numpy() for r in range(world)]
    for d in decs:
        d.close()
    return flags, total, res, transfers.cpu().numpy()


def thin(cuts, size, world):
    """the corpus' cuts thinned out (or filled up) to `world` pieces"""
    inner = cuts[1:-1]
    if len(inner) >= world - 1:
        inner = [inner[i * len(inner) // (world - 1)] for i in range(world - 1)]
    else:
        inner = inner + [size // 256 * (i + 1) // world * 256 for i in range(world - 1 - len(inner))]
    return [0] + sorted(set(inner)) + [size]


def check_pieces(torch, lib, data, cuts, pieces, tr):
    """pieces decode to the shards at `cuts` with verdict 0, and the composed transfers are the traced automaton at every cut"""
    from density_b200 import sharded as S
    shards = [data[a:b] for a, b in zip(cuts[:-1], cuts[1:])]
    flags, total, outs, T = decode_prot_pieces(torch, lib, pieces, [max(s.size, 4) for s in shards])
    assert flags == 0 and total == data.size, cuts
    for r, s in enumerate(shards):
        assert outs[r].size == s.size and (outs[r] == s).all(), (cuts, r)
    for r in range(1, len(cuts) - 1):
        b = cuts[r] // 256
        want = S.decode_prot_candidate(tr.state[b], tr.counter[b] % 16)
        assert S.compose_decode_prot_transfers(T, r) == want, (cuts, r)
    return outs


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_pieces_of_the_protected_encoder_and_slices_of_one_stream(torch_cuda, lib, world):
    from test_gpu_sharded_loopback import _protected_corpora
    import test_gpu_sharded_protected_encode as E
    for data, corpus_cuts in _protected_corpora():
        cuts = thin(corpus_cuts, data.size, world)
        want = oracle.encode("chameleon", data)
        tr = P.trace("chameleon", want, data.size)
        pieces, (eflags, _, _), _, _ = E.encode_prot_shards(torch_cuda, lib, data, cuts)
        assert eflags == 0
        check_pieces(torch_cuda, lib, data, cuts, pieces, tr)
        offs = [int(tr.off[c // 256]) for c in cuts[:-1]] + [want.size]
        slices = [want[a:b] for a, b in zip(offs[:-1], offs[1:])]
        outs = check_pieces(torch_cuda, lib, data, cuts, slices, tr)
        assert (np.concatenate(outs) == oracle.decode("chameleon", want, data.size)).all()


def test_quiet_text_gives_the_pieces_of_decode_sharded(torch_cuda, lib):
    from density_b200 import sharded as S
    data = E_text(3 * MIB + 11)
    want = oracle.encode("chameleon", data)
    tr = P.trace("chameleon", want, data.size)
    assert not tr.copied.any()
    cuts = [0, 4097 * 256, 8000 * 256, data.size]
    offs = [int(tr.off[c // 256]) for c in cuts[:-1]] + [want.size]
    pieces = [want[a:b] for a, b in zip(offs[:-1], offs[1:])]
    outs = check_pieces(torch_cuda, lib, data, cuts, pieces, tr)
    st = ctypes.c_void_p(torch_cuda.cuda.current_stream().cuda_stream)
    decs = [S.ShardedChameleonDecoder() for _ in pieces]
    ins = [torch_cuda.from_numpy(p.copy()).cuda() for p in pieces]
    tables = torch_cuda.empty((len(pieces), S.TABLE_ENTRIES), dtype=torch_cuda.int32, device="cuda")
    for r, d in enumerate(decs):
        assert lib.density_b200_decode_shard_phase1(d._h, ins[r].data_ptr(), ins[r].numel(), outs[r].size, int(r == len(pieces) - 1),
                                                    tables[r].data_ptr(), st) == 0
    for r, d in enumerate(decs):
        carry = S.fold_tables(tables, r).contiguous()
        o = torch_cuda.zeros(outs[r].size + 64, dtype=torch_cuda.uint8, device="cuda")
        sz = torch_cuda.zeros(1, dtype=torch_cuda.int64, device="cuda")
        w = torch_cuda.zeros(8, dtype=torch_cuda.int32, device="cuda")
        assert lib.density_b200_decode_shard_phase2(d._h, carry.data_ptr(), o.data_ptr(), sz.data_ptr(), w.data_ptr(), st) == 0
        torch_cuda.cuda.synchronize()
        assert int(w[2].item()) == 0 and int(sz.item()) == outs[r].size
        assert (o[:outs[r].size].cpu().numpy() == outs[r]).all()
        d.close()


def E_text(n):
    from density_b200 import synth
    return synth.synth_text(n).numpy()


def test_a_cut_off_a_block_boundary_and_a_short_cap_are_refused(torch_cuda, lib):
    data = E_text(2 * MIB)
    data[MIB - 4096:MIB + 4096] = payload("random", 8192, 3)
    want = oracle.encode("chameleon", data)
    tr = P.trace("chameleon", want, data.size)
    assert tr.copied.any()
    cuts = [0, MIB // 256 - 3, MIB // 256 + 5, len(tr.off)]
    offs = [int(tr.off[b]) for b in cuts[:-1]] + [want.size]
    caps = [(cuts[1] - cuts[0]) * 256, (cuts[2] - cuts[1]) * 256, data.size - cuts[2] * 256]
    for delta in (2, -2):
        o = list(offs)
        o[1] += delta
        pieces = [want[a:b] for a, b in zip(o[:-1], o[1:])]
        flags, _, _, _ = decode_prot_pieces(torch_cuda, lib, pieces, [c + 1024 for c in caps])
        assert flags != 0, delta
    pieces = [want[a:b] for a, b in zip(offs[:-1], offs[1:])]
    flags, total, outs, _ = decode_prot_pieces(torch_cuda, lib, pieces, caps)
    assert flags == 0 and total == data.size and (np.concatenate(outs) == data).all()
    for r in range(3):
        short = list(caps)
        short[r] -= 256
        flags, _, _, _ = decode_prot_pieces(torch_cuda, lib, pieces, short)
        assert flags != 0, r


def test_phases_out_of_order_are_refused(torch_cuda, lib):
    from density_b200 import sharded as S
    d = S.ShardedChameleonDecoder()
    t = torch_cuda.zeros(S.DECODE_PROT_TRANSFER_WORDS * 2, dtype=torch_cuda.int32, device="cuda")
    tab = torch_cuda.zeros(S.TABLE_ENTRIES, dtype=torch_cuda.int32, device="cuda")
    st = ctypes.c_void_p(torch_cuda.cuda.current_stream().cuda_stream)
    assert lib.density_b200_decode_shard_prot_phase1(d._h, t.data_ptr(), 2, 1, tab.data_ptr(), st) != 0
    assert lib.density_b200_decode_shard_prot_phase2(d._h, None, None, t.data_ptr(), t.data_ptr(), st) != 0
    d.close()
