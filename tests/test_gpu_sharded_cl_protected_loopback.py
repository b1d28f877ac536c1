"""density_b200_encode_sharded_cl_protected at W = 2..8 ranks on one H100 (pytest -m gpu), through the loopback collective library of
test_gpu_sharded_loopback.py: the pieces equal the oracle's stream on mixed data, noise and text with noise bursts at ragged cuts, every
rank reaches the same verdict, every gather root receives the stream, a budget that is too small is refused on every rank, bad
arguments return before any collective, and every rank issues the collectives include/density_b200.h lists for the driver."""
import numpy as np
import pytest

import oracle
from test_gpu_sharded_loopback import (ALG, CANARY, EARG, OK, Ranks, _p, ag, check_logs, cut, env, same, text)  # noqa: F401
from conftest import payload

pytestmark = pytest.mark.gpu

MIB = 1 << 20


def encode(env, alg, shards, gather_root=-1):
    """One density_b200_encode_sharded_cl_protected of `shards` on fresh handles, with the per-call checks. Returns (rc, flags, total,
    pieces, gathered)."""
    torch, lib, _ = env
    W = len(shards)
    safe = getattr(lib, f"{alg}_safe_encode_buffer_size")
    caps = [safe(s.size) for s in shards]
    d_in = [torch.from_numpy(s.copy()).cuda() if s.size else None for s in shards]
    d_out = [torch.full((c + 64,), CANARY, dtype=torch.uint8, device="cuda") for c in caps]
    d_sz = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    d_fl = [torch.full((1,), -1, dtype=torch.int32, device="cuda") for _ in range(W)]
    d_tot = [torch.full((1,), -1, dtype=torch.int64, device="cuda") for _ in range(W)]
    gcap = sum(caps)
    d_g = torch.full((gcap + 64,), CANARY, dtype=torch.uint8, device="cuda") if gather_root >= 0 else None

    def call(r, h, st):
        g = (_p(d_g), gcap) if r == gather_root else (None, 0)
        return lib.density_b200_encode_sharded_cl_protected(h, ALG[alg], _p(d_in[r]), shards[r].size, _p(d_out[r]), caps[r], _p(d_sz[r]),
                                                            _p(d_fl[r]), _p(d_tot[r]), gather_root, *g, st)

    with Ranks(env, W) as R:
        res = R.run(call)
        rc = same([x[0] for x in res], "rc")
        assert rc == OK, res
        for r in range(W):
            assert bool((d_out[r][caps[r]:] == CANARY).all()), f"rank {r} wrote past cap"
        if d_g is not None:
            assert bool((d_g[gcap:] == CANARY).all()), "the gather wrote past gather_cap"
        flags = same([int(f.item()) for f in d_fl], "flags")
        total = same([int(t.item()) for t in d_tot], "total")
        sizes = [int(s.item()) for s in d_sz]
        pieces = [d_out[r][:sizes[r]].cpu().numpy() for r in range(W)]
        wp, wc = lib.density_b200_cl_table_words(ALG[alg], 0), lib.density_b200_cl_table_words(ALG[alg], 1)
        want = ag(2, 8) + ag(wp, wc, 200, 8) * lib.density_b200_prot_round_budget() + ag(8)
        check_logs(R, want, sizes, gather_root if not flags else -1)
        gathered = d_g[:total].cpu().numpy() if d_g is not None and not flags else None
    return flags, total, pieces, gathered


def corpora():
    """mixed data, noise, and text with noise bursts that end at, straddle and start at a cut"""
    from density_b200 import synth
    out = [synth.synth_mixed(2 * MIB).numpy()[:2 * MIB - 3], payload("random", MIB + 77, 2)]
    data = text(2 * MIB, first_page=5)
    rnd = payload("random", 64 * 1024, 7)
    for i, b in enumerate([1000, 2501, 4097]):
        lo = [b * 256 - 2048, b * 256 - 1024, b * 256][i]
        data[lo:lo + 2048] = rnd[i * 8192:i * 8192 + 2048]
    out.append(data)
    return out


def ragged_cuts(n, world, seed):
    rng = np.random.default_rng(seed)
    body = n // 256
    inner = sorted(int(v) for v in rng.choice(np.arange(1, body), world - 1, replace=False))
    return [0] + [256 * u for u in inner] + [n]


@pytest.mark.parametrize("alg", ["cheetah", "lion"])
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_encode_sharded_cl_protected(env, alg, world):
    for k, data in enumerate(corpora()):
        cuts = ragged_cuts(data.size, world, 10 * world + k)
        if k == 2:
            cuts = sorted(set(cuts[:-1] + [1000 * 256, 2501 * 256]))[:world] + [data.size]
        want = oracle.encode(alg, data)
        root = [-1, 0, world - 1][k]
        flags, total, pieces, gathered = encode(env, alg, cut(data, cuts), root)
        assert flags == 0 and total == want.size, (alg, world, k)
        assert (np.concatenate(pieces) == want).all(), (alg, world, k)
        if root >= 0:
            assert (gathered == want).all()


def test_encode_sharded_cl_protected_empty_first_rank_and_every_root(env):
    from density_b200 import synth
    data = synth.synth_mixed(MIB).numpy()
    for alg in ("cheetah", "lion"):
        want = oracle.encode(alg, data)
        cuts = [0, 0, 1001 * 256, 1001 * 256, data.size]
        for root in range(4):
            flags, total, _, gathered = encode(env, alg, cut(data, cuts), root)
            assert flags == 0 and total == want.size and (gathered == want).all(), (alg, root)


def test_encode_sharded_cl_protected_budget_too_small_is_refused(env):
    _, lib, _ = env
    data = payload("random", MIB, 4)
    lib.density_b200_test_set_prot_rounds(1)
    try:
        for alg in ("cheetah", "lion"):
            flags, total, pieces, _ = encode(env, alg, cut(data, [0, 1001 * 256, 2002 * 256, data.size]), gather_root=1)
            assert flags != 0 and total == 0 and all(p.size == 0 for p in pieces)
    finally:
        lib.density_b200_test_set_prot_rounds(0)


def test_encode_sharded_cl_protected_bad_arguments_before_any_collective(env):
    torch, lib, _ = env
    d_in = torch.from_numpy(text(MIB)).cuda()
    cap = lib.cheetah_safe_encode_buffer_size(MIB)
    d_out = torch.zeros(cap + 8, dtype=torch.uint8, device="cuda")
    s = [torch.zeros(2, dtype=torch.int64, device="cuda") for _ in range(3)]
    fn = lib.density_b200_encode_sharded_cl_protected
    with Ranks(env, 2) as R:
        bad = [
            lambda h, st: fn(h, 0, d_in.data_ptr(), MIB, d_out.data_ptr(), cap, s[0].data_ptr(), s[1].data_ptr(), s[2].data_ptr(), -1, None, 0, st),
            lambda h, st: fn(h, 1, d_in.data_ptr(), MIB, d_out.data_ptr(), cap, s[0].data_ptr(), s[1].data_ptr(), s[2].data_ptr(), 1, None, 0, st),
            lambda h, st: fn(h, 1, d_in.data_ptr() + 1, MIB - 4, d_out.data_ptr(), cap, s[0].data_ptr(), s[1].data_ptr(), s[2].data_ptr(), -1,
                             None, 0, st),
            lambda h, st: fn(h, 2, d_in.data_ptr(), MIB, d_out.data_ptr(), cap, s[0].data_ptr() + 4, s[1].data_ptr(), s[2].data_ptr(), -1,
                             None, 0, st),
            lambda h, st: fn(h, 2, d_in.data_ptr(), MIB, d_out.data_ptr(), cap, s[0].data_ptr(), s[1].data_ptr(), s[2].data_ptr() + 4, -1,
                             None, 0, st),
        ]
        for f in bad:
            res = R.run(lambda r, h, st: f(h, st), ranks=[1])
            assert res[0][0] == EARG, res
            assert R.logs([1]) == [[]]
