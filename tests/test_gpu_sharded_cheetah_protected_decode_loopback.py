"""density_b200_decode_sharded_cheetah_protected at W = 2, 3, 4 and 8 ranks on one H100 (pytest -m gpu), through the loopback collective
library of test_gpu_sharded_loopback.py: the pieces of density_b200_encode_sharded_cl_protected (Cheetah) decode back to their shards on
every rank with one verdict, nothing is written past cap, a short cap on one rank is refused on every rank, and every rank issues the
driver's collectives: the transfers, the chunk-map transfers, the prediction transfers and round words of every round, the seam words."""
import numpy as np
import pytest

from test_gpu_sharded_loopback import CANARY, OK, Ranks, _p, ag, check_logs, cut, env, same  # noqa: F401
from test_gpu_sharded_cl_protected_loopback import corpora, encode, ragged_cuts

pytestmark = pytest.mark.gpu

MIB_HALF = 1 << 19


def decode_protected(env, pieces, caps):
    """density_b200_decode_sharded_cheetah_protected of `pieces` on fresh handles. Returns (flags, total, outs)."""
    torch, lib, _ = env
    W = len(pieces)
    d_in = [torch.from_numpy(np.ascontiguousarray(p)).cuda() if p.size else None for p in pieces]
    d_out = [torch.full((c + 64,), CANARY, dtype=torch.uint8, device="cuda") for c in caps]
    d_sz = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    d_fl = [torch.full((1,), -1, dtype=torch.int32, device="cuda") for _ in range(W)]
    d_tot = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    fn = lib.density_b200_decode_sharded_cheetah_protected
    with Ranks(env, W) as R:
        res = R.run(lambda r, h, st: fn(h, _p(d_in[r]), pieces[r].size, _p(d_out[r]), caps[r], _p(d_sz[r]), _p(d_fl[r]), _p(d_tot[r]), st))
        assert same([x[0] for x in res], "rc") == OK, res
        for r in range(W):
            assert bool((d_out[r][caps[r]:] == CANARY).all()), f"rank {r} wrote past cap"
        flags = same([int(f.item()) for f in d_fl], "flags")
        total = same([int(t.item()) for t in d_tot], "total")
        want = ag(3200, lib.density_b200_cheetah_cmap_words()) + ag(131072, 4) * lib.density_b200_cheetah_decode_round_budget() + ag(8)
        check_logs(R, want)
        outs = [d_out[r][:max(int(d_sz[r].item()), 0)].cpu().numpy() for r in range(W)]
    return flags, total, outs


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_decode_sharded_cheetah_protected_pieces_of_the_protected_encoder(env, world):
    for k, data in enumerate(corpora()):
        shards = cut(data, ragged_cuts(data.size, world, 10 * world + k))
        flags, _, pieces, _ = encode(env, "cheetah", shards)
        assert flags == 0
        flags, total, outs = decode_protected(env, pieces, [max(s.size, 4) for s in shards])
        assert flags == 0 and total == data.size
        for r, s in enumerate(shards):
            assert outs[r].size == s.size and (outs[r] == s).all(), (world, k, r)


def test_decode_sharded_cheetah_protected_empty_first_rank_and_a_short_cap(env):
    """an empty rank 0 (the stream start on rank 1) decodes; a cap 128 bytes short on one rank is refused on every rank"""
    data = corpora()[0][:MIB_HALF]
    shards = cut(data, [0, 0, 1111 * 256, data.size])
    flags, _, pieces, _ = encode(env, "cheetah", shards)
    assert flags == 0
    caps = [max(s.size, 4) for s in shards]
    flags, total, outs = decode_protected(env, pieces, caps)
    assert flags == 0 and total == data.size and (np.concatenate(outs) == data).all()
    for r in (1, 2):
        short = list(caps)
        short[r] -= 128
        flags, _, _ = decode_protected(env, pieces, short)
        assert flags != 0, r

