"""density_b200_decode_sharded_stream_protected and density_b200_decode_sharded_cheetah_stream_protected at W = 2, 3, 5 and 8 ranks on one
H100 (pytest -m gpu), through the loopback collective library of test_gpu_sharded_loopback.py: streams with copy-mode blocks, cut at byte
ranges, decode back to the original on every rank with one verdict and the output offsets of the pieces, nothing is written past cap,
a refused composition is refused on every rank after the maps' all-gather alone, and every rank issues the collectives the header
lists in that order."""
import numpy as np
import pytest

import prot_locate_model as L
from test_gpu_sharded_loopback import CANARY, OK, Ranks, _p, ag, check_logs, env, same  # noqa: F401
from test_gpu_sharded_stream_protected_decode import corpus

pytestmark = pytest.mark.gpu


def decode_stream_protected(env, alg, stream, lay, caps=None):
    """The driver on every rank of a layout [(offset, n_range, n_halo)] of a stream whose composition locates every piece (no 0xFFFF /
    0xFFFE on the path). Returns (flags, total, outs, offsets); checks the logs: the maps' all-gather, then every collective of the
    located piece's path, on every rank."""
    torch, lib, _ = env
    W = len(lay)
    caps = caps or [(2 if alg == "chameleon" else 16) * (n + h) for _, n, h in lay]
    d_in = [torch.from_numpy(np.ascontiguousarray(stream[o:o + n + h])).cuda() if n + h else None for o, n, h in lay]
    d_out = [torch.full((c + 64,), CANARY, dtype=torch.uint8, device="cuda") for c in caps]
    d_sz = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    d_off = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    d_fl = [torch.full((1,), -1, dtype=torch.int32, device="cuda") for _ in range(W)]
    d_tot = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    fn = lib.density_b200_decode_sharded_stream_protected if alg == "chameleon" else lib.density_b200_decode_sharded_cheetah_stream_protected
    with Ranks(env, W) as R:
        res = R.run(lambda r, h, st: fn(h, _p(d_in[r]), lay[r][1], lay[r][2], _p(d_out[r]), caps[r], _p(d_sz[r]), _p(d_off[r]), _p(d_fl[r]),
                                        _p(d_tot[r]), st))
        assert same([x[0] for x in res], "rc") == OK, res
        for r in range(W):
            assert bool((d_out[r][caps[r]:] == CANARY).all()), f"rank {r} wrote past cap"
        flags = same([int(f.item()) for f in d_fl], "flags")
        total = same([int(t.item()) for t in d_tot], "total")
        want = ag(L.map_words(alg))
        if alg == "chameleon":
            want += ag(65536, 8)
        else:
            want += ag(lib.density_b200_cheetah_cmap_words()) + ag(131072, 4) * lib.density_b200_cheetah_decode_round_budget() + ag(8)
        check_logs(R, want)
        outs = [d_out[r][:max(int(d_sz[r].item()), 0)].cpu().numpy() for r in range(W)]
        offsets = [int(o.item()) for o in d_off]
    return flags, total, outs, offsets


@pytest.mark.parametrize("alg", ["chameleon", "cheetah"])
@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_streams_with_copy_mode_decode_on_every_rank(env, alg, world):
    from density_b200 import sharded as S
    for name in ("noise", "synth_mixed", "text_bursts"):
        data, s = corpus(name, alg)
        flags, total, outs, offsets = decode_stream_protected(env, alg, s, S.stream_ranges(s.size, world))
        assert flags == 0 and total == data.size, (name, world)
        for r in range(world):
            assert (outs[r] == data[offsets[r]:offsets[r] + outs[r].size]).all(), (name, r)
        assert (np.concatenate(outs) == data).all()


@pytest.mark.parametrize("alg", ["chameleon", "cheetah"])
def test_empty_ranks_and_a_short_cap(env, alg):
    data, s = corpus("noise", alg)
    U = L.RANGE_UNIT
    lay = L.layout(s.size, [0, 9 * U, 0, 30 * U, None])
    flags, total, outs, _ = decode_stream_protected(env, alg, s, lay)
    assert flags == 0 and total == data.size and (np.concatenate(outs) == data).all()
    caps = [max(o.size, 4) for o in outs]
    r = int(np.argmax([o.size for o in outs]))
    caps[r] -= 1
    flags, _, _, _ = decode_stream_protected(env, alg, s, lay, caps)
    assert flags != 0


def test_a_bad_layout_is_refused_alike_on_every_rank(env):
    """a halo that is not min(264, the later bytes) on one rank: every rank returns DENSITY_B200_EARG after the maps' all-gather"""
    torch, lib, _ = env
    _, s = corpus("noise", "chameleon")
    U = L.RANGE_UNIT
    lay = [(0, 4 * U, 100), (4 * U, s.size - 4 * U, 0)]
    d_in = [torch.from_numpy(np.ascontiguousarray(s[o:o + n + h])).cuda() for o, n, h in lay]
    d_out = [torch.zeros(2 * (n + h), dtype=torch.uint8, device="cuda") for _, n, h in lay]
    d_sz = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in lay]
    d_fl = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in lay]
    fn = lib.density_b200_decode_sharded_stream_protected
    with Ranks(env, 2) as R:
        res = R.run(lambda r, h, st: fn(h, _p(d_in[r]), lay[r][1], lay[r][2], _p(d_out[r]), d_out[r].numel(), _p(d_sz[r]), None, _p(d_fl[r]),
                                        None, st))
        assert same([x[0] for x in res], "rc") == 4
        check_logs(R, ag(L.map_words("chameleon")))
