"""density_b200_decode_sharded_protected at W = 2..8 ranks on one H100 (pytest -m gpu), through the loopback collective library of
test_gpu_sharded_loopback.py: the pieces of density_b200_encode_sharded_protected decode back to their shards on every rank with one
verdict, nothing is written past cap, and every rank issues the driver's collectives: the transfers, the tables, the seam words."""
import numpy as np
import pytest

from test_gpu_sharded_loopback import (CANARY, OK, Ranks, _p, _protected_corpora, ag, check_logs, cut, encode, env, same,  # noqa: F401
                                       text)
from conftest import splitmix_bytes

pytestmark = pytest.mark.gpu


def decode_protected(env, pieces, caps):
    """density_b200_decode_sharded_protected of `pieces` on fresh handles. Returns (flags, total, outs)."""
    torch, lib, _ = env
    W = len(pieces)
    d_in = [torch.from_numpy(np.ascontiguousarray(p)).cuda() if p.size else None for p in pieces]
    d_out = [torch.full((c + 64,), CANARY, dtype=torch.uint8, device="cuda") for c in caps]
    d_sz = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    d_fl = [torch.full((1,), -1, dtype=torch.int32, device="cuda") for _ in range(W)]
    d_tot = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    with Ranks(env, W) as R:
        res = R.run(lambda r, h, st: lib.density_b200_decode_sharded_protected(h, _p(d_in[r]), pieces[r].size, _p(d_out[r]), caps[r],
                                                                               _p(d_sz[r]), _p(d_fl[r]), _p(d_tot[r]), st))
        assert same([x[0] for x in res], "rc") == OK, res
        for r in range(W):
            assert bool((d_out[r][caps[r]:] == CANARY).all()), f"rank {r} wrote past cap"
        flags = same([int(f.item()) for f in d_fl], "flags")
        total = same([int(t.item()) for t in d_tot], "total")
        check_logs(R, ag(3200) + ag(65536) + ag(8))
        outs = [d_out[r][:max(int(d_sz[r].item()), 0)].cpu().numpy() for r in range(W)]
    return flags, total, outs


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_decode_sharded_protected_pieces_of_the_protected_encoder(env, world):
    for data, cuts in _protected_corpora():
        inner = cuts[1:-1]
        if len(inner) >= world - 1:
            inner = [inner[i * len(inner) // (world - 1)] for i in range(world - 1)]
        else:
            inner = inner + [data.size // 256 * (i + 1) // world * 256 for i in range(world - 1 - len(inner))]
        shards = cut(data, [0] + sorted(inner) + [data.size])
        o = encode(env, "chameleon", shards, "protected")
        assert o["rc"] == OK and o["flags"] == 0
        flags, total, outs = decode_protected(env, o["pieces"], [max(s.size, 4) for s in shards])
        assert flags == 0 and total == data.size
        for r, s in enumerate(shards):
            assert outs[r].size == s.size and (outs[r] == s).all(), (world, r)


def test_decode_sharded_protected_copy_mode_piece_and_a_short_cap(env):
    """the pieces decode_sharded refuses decode here; a short cap on one rank is refused on every rank"""
    d = text(2 * (1 << 20), first_page=6)
    d[(1 << 20) + 4096:(1 << 20) + 4096 + 64 * 1024] = splitmix_bytes(64 * 1024, 8)
    shards = cut(d, [0, 1 << 20, d.size])
    o = encode(env, "chameleon", shards, "protected")
    assert o["rc"] == OK and o["flags"] == 0
    flags, total, outs = decode_protected(env, o["pieces"], [s.size for s in shards])
    assert flags == 0 and total == d.size and (np.concatenate(outs) == d).all()
    flags, _, _ = decode_protected(env, o["pieces"], [shards[0].size, shards[1].size - 256])
    assert flags != 0
