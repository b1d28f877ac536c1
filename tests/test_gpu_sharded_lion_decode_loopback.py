"""density_b200_decode_sharded_lion and _protected at W = 2..8 ranks on one H100 (pytest -m gpu), through the loopback collective library
of test_gpu_sharded_loopback.py: the pieces of the sharded Lion encoders decode back to their shards on every rank with one verdict,
nothing is written past cap, a short cap on one rank is refused on every rank, and every rank issues the driver's collectives in the
order the header states: [the transfers,] the chunk-map transfers, the walk's state received from rank - 1, the state sent to rank + 1,
the seam words."""
import numpy as np
import pytest

import loopback as lb
from test_gpu_sharded_loopback import CANARY, OK, Ranks, _p, ag, check_logs, cut, env, same  # noqa: F401
from test_gpu_sharded_cl_protected_loopback import corpora, encode, ragged_cuts
from test_gpu_sharded_loopback import encode as encode_plain

pytestmark = pytest.mark.gpu

STATE_WORDS = 5 * 65536 + 8          # DENSITY_B200_LION_STATE_WORDS
MIB_HALF = 1 << 19


def decode(env, pieces, caps, prot):
    """density_b200_decode_sharded_lion(_protected) of `pieces` on fresh handles. Returns (flags, total, outs)."""
    torch, lib, _ = env
    W = len(pieces)
    d_in = [torch.from_numpy(np.ascontiguousarray(p)).cuda() if p.size else None for p in pieces]
    d_out = [torch.full((c + 64,), CANARY, dtype=torch.uint8, device="cuda") for c in caps]
    d_sz = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    d_fl = [torch.full((1,), -1, dtype=torch.int32, device="cuda") for _ in range(W)]
    d_tot = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    fn = lib.density_b200_decode_sharded_lion_protected if prot else lib.density_b200_decode_sharded_lion
    with Ranks(env, W) as R:
        res = R.run(lambda r, h, st: fn(h, _p(d_in[r]), pieces[r].size, _p(d_out[r]), caps[r], _p(d_sz[r]), _p(d_fl[r]), _p(d_tot[r]), st))
        assert same([x[0] for x in res], "rc") == OK, res
        for r in range(W):
            assert bool((d_out[r][caps[r]:] == CANARY).all()), f"rank {r} wrote past cap"
        flags = same([int(f.item()) for f in d_fl], "flags")
        total = same([int(t.item()) for t in d_tot], "total")
        head = ag(3200) if prot else []
        for r, log in enumerate(R.logs()):
            want = head + ag(lib.density_b200_cheetah_cmap_words())
            if r > 0:
                want += [(lb.RECV, STATE_WORDS, lb.UINT32, r - 1)]
            if r < W - 1:
                want += [(lb.SEND, STATE_WORDS, lb.UINT32, r + 1)]
            want += ag(8)
            assert log == want, (r, log, want)
        outs = [d_out[r][:max(int(d_sz[r].item()), 0)].cpu().numpy() for r in range(W)]
    return flags, total, outs


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_decode_sharded_lion_pieces_of_the_encoder(env, world):
    from density_b200 import synth
    data = synth.synth_text(MIB_HALF * 3, first_page=world).numpy()
    step = data.size // world // 256 * 256        # uneven shards, all cut behind the copy run of the stream start
    shards = cut(data, [0] + [step * k + 256 * (k % 3) for k in range(1, world)] + [data.size])
    r = encode_plain(env, "lion", shards, driver="cl")
    assert r["flags"] == 0
    flags, total, outs = decode(env, r["pieces"], [max(s.size, 4) for s in shards], prot=False)
    assert flags == 0 and total == data.size
    for k, s in enumerate(shards):
        assert outs[k].size == s.size and (outs[k] == s).all(), (world, k)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_decode_sharded_lion_protected_pieces_of_the_protected_encoder(env, world):
    for k, data in enumerate(corpora()):
        data = data[:MIB_HALF * 2 + 77]
        shards = cut(data, ragged_cuts(data.size, world, 10 * world + k))
        flags, _, pieces, _ = encode(env, "lion", shards)
        assert flags == 0
        flags, total, outs = decode(env, pieces, [max(s.size, 4) for s in shards], prot=True)
        assert flags == 0 and total == data.size
        for r, s in enumerate(shards):
            assert outs[r].size == s.size and (outs[r] == s).all(), (world, k, r)


def test_decode_sharded_lion_protected_empty_first_rank_and_a_short_cap(env):
    """an empty rank 0 (the stream start on rank 1) decodes; a cap 64 bytes short on one rank is refused on every rank"""
    data = corpora()[0][:MIB_HALF]
    shards = cut(data, [0, 0, 1111 * 256, data.size])
    flags, _, pieces, _ = encode(env, "lion", shards)
    assert flags == 0
    caps = [max(s.size, 4) for s in shards]
    flags, total, outs = decode(env, pieces, caps, prot=True)
    assert flags == 0 and total == data.size and (np.concatenate(outs) == data).all()
    for r in (1, 2):
        short = list(caps)
        short[r] -= 64
        flags, _, _ = decode(env, pieces, short, prot=True)
        assert flags != 0, r
