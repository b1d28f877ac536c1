"""Sharded Lion decode of streams with copy-mode blocks, through the phase API on one device (needs an H100: pytest -m gpu).

W pieces run density_b200_lion_decode_shard_prot_transfer / _prot_phase1, then phase 2, the walk and phase 3, the exchanges replaced by
stacking the transfers and chunk-map tables and the relay by one device buffer. Whatever the data -- noise, synth_mixed, text with noise
bursts at and across the cuts, the seam cases of every automaton state -- every piece of the protected sharded Lion encoder, and every
slice of one lion_encode stream at the same prefix sums, decodes to its shard byte for byte with verdict 0, and the composed transfers
are the in-order automaton of the stream at every cut."""
import numpy as np
import pytest

from conftest import payload, splitmix_bytes
from test_gpu_sharded_lion_decode import (ALG, BS, MIB, _enc_and_cuts, check_data, decode_lion_pieces, lib, single_counts, slices, text,  # noqa: F401
                                          torch_cuda, trace_of)

pytestmark = pytest.mark.gpu


def check_transfers(torch, lib, data, cuts):
    """the slices of the oracle's stream decode with verdict 0 and their composed transfers are the traced automaton at every cut"""
    from density_b200 import sharded as S
    enc, tr = trace_of(data)
    shards = [data[a:b] for a, b in zip(cuts[:-1], cuts[1:])]
    flags, total, outs, _, _, T = decode_lion_pieces(torch, lib, slices(enc, tr, cuts), [max(s.size, 4) for s in shards], prot=True)
    assert flags == 0 and total == data.size and (np.concatenate(outs) == data).all(), cuts
    for r in range(1, len(cuts) - 1):
        if cuts[r] == data.size:
            continue
        b = cuts[r] // BS
        assert S.compose_decode_prot_transfers(T, r) == S.decode_prot_candidate(tr.state[b], tr.counter[b] % 16), (cuts, r)


def cuts_at(n, *units):
    return [0] + [u * 256 for u in units] + [n]


def test_noise_mixed_and_text(torch_cuda, lib):
    from density_b200 import synth
    for data in (payload("random", MIB // 2 + 77, 1), synth.synth_mixed(MIB).numpy(), text(MIB + 3, first_page=3)):
        n = data.size
        check_data(torch_cuda, lib, data, cuts_at(n, 411, 1003, 1501), prot=True)
        check_transfers(torch_cuda, lib, data, cuts_at(n, *range(197, n // 256, n // 256 // 8)))


def test_noise_bursts_at_and_across_cuts(torch_cuda, lib):
    data = text(MIB, first_page=2)
    rnd = payload("random", 64 * 1024, 7)
    cuts_b = [500, 1251, 2049, 3000]
    for i, b in enumerate(cuts_b):          # a burst ending at the cut, one straddling it, one starting at it, one across
        lo = [b * 256 - 2048, b * 256 - 1024, b * 256, b * 256 - 512][i]
        ln = [2048, 2048, 4096, 768][i]
        data[lo:lo + ln] = rnd[i * 8192:i * 8192 + ln]
    check_data(torch_cuda, lib, data, cuts_at(data.size, *cuts_b), prot=True)
    check_transfers(torch_cuda, lib, data, cuts_at(data.size, *cuts_b))


def test_empty_pieces_and_a_tiny_last_piece(torch_cuda, lib):
    from density_b200 import synth
    d = synth.synth_mixed(MIB).numpy()[:200 * 1024 + 3]
    n, nb = d.size, d.size // 256
    for cuts in ([0, 0, 0, 300 * 256, n],                      # the stream start in piece 2, behind two empty pieces
                 [0, 100 * 256, 100 * 256, 100 * 256, n],       # empty middle pieces
                 [0, 256, 512, 768, 1024, nb * 256, n]):        # 256-byte shards, and a last piece shorter than one block
        check_data(torch_cuda, lib, d, cuts, encoder=cuts[1] > 0, prot=True)


def test_every_seam_case_is_accepted(torch_cuda, lib):
    from test_gpu_protection import _shard_cases
    n = 0
    for end, nxt, cut, bld in _shard_cases(ALG):
        data, _ = bld.realize()
        check_transfers(torch_cuda, lib, data, [0, cut, data.size])
        n += 1
    assert n >= 20


def test_the_quiet_paths_refusals_are_accepted(torch_cuda, lib):
    torch = torch_cuda
    t = text(2 * MIB, first_page=5)
    noise = splitmix_bytes(MIB, 12)
    cases = []
    d = np.concatenate([t[:MIB], noise[:256 * 1024], t[MIB:]])          # copy mode in piece 1
    cases.append((d, [0, MIB - 64 * 1024, d.size]))
    d = t.copy()                                                          # an incompressible block on each side of the cut
    d[MIB - 64:MIB + 64] = noise[:128]
    cases.append((d, [0, MIB, d.size]))
    d = t.copy()                                                          # piece 0 ends with a copy penalty pending
    d[MIB - 128:MIB] = noise[:128]
    cases.append((d, [0, MIB, d.size]))
    d = np.concatenate([t[:MIB], noise[:64 * 1024], t[MIB:]])            # piece 0 ends inside a copy run
    cases.append((d, [0, MIB + 64 * 1024, d.size]))
    for d, cuts in cases:
        enc, pc = _enc_and_cuts(d, cuts)
        pieces = [enc[a:b] for a, b in zip(pc[:-1], pc[1:])]
        flags, total, outs, _, _, _ = decode_lion_pieces(torch, lib, pieces, [cuts[1], d.size - cuts[1]], prot=True)
        assert flags == 0 and total == d.size and (np.concatenate(outs) == d).all(), cuts


def test_a_moved_cut_and_a_short_cap_are_refused(torch_cuda, lib):
    torch = torch_cuda
    data = text(MIB)
    data[MIB // 2 - 4096:MIB // 2 + 4096] = payload("random", 8192, 3)
    enc, tr = trace_of(data)
    assert tr.copied.any()
    cuts = [0, MIB // 2 - 3 * BS, MIB // 2 + 5 * BS, data.size]
    offs = [int(tr.off[c // BS]) for c in cuts[:-1]] + [enc.size]
    caps = [b - a for a, b in zip(cuts[:-1], cuts[1:])]
    for delta in (2, -2):
        o = list(offs)
        o[1] += delta
        flags, _, _, _, _, _ = decode_lion_pieces(torch, lib, [enc[a:b] for a, b in zip(o[:-1], o[1:])], [c + 1024 for c in caps], prot=True)
        assert flags != 0, delta
    pieces = [enc[a:b] for a, b in zip(offs[:-1], offs[1:])]
    flags, total, outs, _, _, _ = decode_lion_pieces(torch, lib, pieces, caps, prot=True)
    assert flags == 0 and total == data.size and (np.concatenate(outs) == data).all()
    for r in range(3):
        short = list(caps)
        short[r] -= 64
        flags, _, _, words, _, _ = decode_lion_pieces(torch, lib, pieces, short, prot=True)
        assert flags != 0 and words[r][2] == 1, r


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
        flags, _, got, _, _, _ = decode_lion_pieces(torch, lib, [e[a:b] for a, b in zip(p[:-1], p[1:])], [16 * e.size + 256] * 2, prot=True)
        if flags == 0:
            want, _ = single_counts(torch, lib, e, 16 * e.size + 256)
            cat = np.concatenate(got)
            assert cat.size == want.size and (cat == want).all(), trial
