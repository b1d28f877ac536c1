"""The copy-map iteration of the sharded Cheetah / Lion encode with copy mode (density_b200_cl_shard_prot_*), modelled on the CPU.

Under a copy map M the in-order model of the encoders drops the copied blocks' quads (they touch neither table nor the context chain),
gives every encoded block its size and its incompressible bit; copied blocks keep the bit of the round before. A round then runs the
automaton shard by shard from the transfers of the shards before it (sharded.compose_prot_transfers), counting blocks from the stream
start. The shard at the stream start starts from its own settled map, the others from the empty map. The settled map must be the one
the oracle's stream shows, the prefix on which the map agrees with it must grow by a block at least every round, and the {has, quad}
words each shard publishes must give every later shard the in-order context of its first encoded quad."""
import numpy as np
import pytest

import oracle
import protection as P
from conftest import GOLDEN_DIR, splitmix_bytes
from density_b200 import sharded as S
from test_sharded_cl_cpu import INV, hf


def block_sizes(alg, data, cm):
    """Encoded size of every block under copy map cm (a copied block: its length) and the last encoded quad before every block
    (None: the stream start)."""
    lion, B = alg == "lion", P.BS[alg]
    nb = (data.size + B - 1) // B
    qs = data[:data.size // 4 * 4].view(np.uint32)
    pred, chunk, ctx, last = {}, {}, 0, None
    sizes, before = [], []
    for b in range(nb):
        before.append(last)
        blen = min(B, data.size - b * B)
        if cm[b]:
            sizes.append(blen)
            continue
        size = (6 if lion else 8) + blen % 4
        for i in range(b * B // 4, (b * B + blen) // 4):
            q = int(qs[i])
            lst = pred.get(ctx, [0] * 5 if lion else 0)
            if lion:
                hit = lst.index(q) if q in lst else None
                pred[ctx] = [q] + (lst[:hit] + lst[hit + 1:] if hit is not None else lst[:4])
            else:
                hit = 0 if lst == q else None
                pred[ctx] = q
            h, f = hf(q)
            if hit is None:
                a, bb = chunk.get(h, (0, 0) if h == 0 else (INV, INV))
                size += 2 if f in (a, bb) else 4
                if f != a:
                    chunk[h] = (f, a)
            ctx, last = h, q
        sizes.append(size)
    return sizes, before


def incompressible(alg, data, sizes):
    B = P.BS[alg]
    return [data.size - b * B >= B and s >= B for b, s in enumerate(sizes)]


def transfer(inc, first_block):
    out = np.zeros(S.PROT_TRANSFER_WORDS, dtype=np.int64)
    for c in range(S.PROT_TRANSFER_WORDS):
        ps = P.Protection(*S.prot_state(c), counter=first_block)
        for bit in inc:
            ps.step(bool(bit))
        out[c] = S.prot_candidate(ps.key())
    return out


def settle_alone(alg, data):
    """The single-device iteration on `data` alone (the staged iteration of the shard at the stream start)."""
    nb = (data.size + P.BS[alg] - 1) // P.BS[alg]
    cm, inc = [False] * nb, [False] * nb
    for _ in range(64):
        sizes, _ = block_sizes(alg, data, cm)
        inc = [i if c else n for c, i, n in zip(cm, inc, incompressible(alg, data, sizes))]
        ps = P.Protection()
        new = [ps.step(bool(bit)) for bit in inc]
        if new == cm:
            return cm
        cm = new
    raise AssertionError("did not settle")


def rounds(alg, data, cuts):
    """The round protocol over shards [cuts[r], cuts[r + 1]) (bytes). Returns the maps M_0, M_1, ... up to the settled one, and per
    round the carried-in {has, quad} of every shard."""
    B = P.BS[alg]
    nb = (data.size + B - 1) // B
    blocks = [c // B for c in cuts[:-1]] + [nb]
    first = next(r for r in range(len(cuts) - 1) if cuts[r + 1] > cuts[r])
    cm = [False] * nb
    cm[:blocks[first + 1]] = settle_alone(alg, data[:cuts[first + 1]])          # the warm start
    inc = [False] * nb
    maps, carried = [list(cm)], []
    for _ in range(32):
        sizes, before = block_sizes(alg, data, cm)
        inc = [i if c else n for c, i, n in zip(cm, inc, incompressible(alg, data, sizes))]
        T = np.stack([transfer(inc[a:b], a) for a, b in zip(blocks[:-1], blocks[1:])])
        new = []
        for r, (a, b) in enumerate(zip(blocks[:-1], blocks[1:])):
            ps = P.Protection(*S.prot_state(S.compose_prot_transfers(T, r)), counter=a)
            new.extend(ps.step(bool(bit)) for bit in inc[a:b])
        # the words each shard publishes under the new map, and what every shard takes from the shards before it
        qs = data[:data.size // 4 * 4].view(np.uint32)
        words = []
        for a, b in zip(blocks[:-1], blocks[1:]):
            enc = [k for k in range(a, b) if not new[k] and k * B // 4 < qs.size]
            words.append((1, int(qs[min((enc[-1] + 1) * B // 4, qs.size) - 1])) if enc else (0, 0))
        ctx = []
        for r in range(len(words)):
            got = [w for w in words[:r] if w[0]]
            ctx.append(got[-1][1] if got else None)
        carried.append((ctx, new))
        maps.append(new)
        if new == cm:
            return maps, carried
        cm = new
    raise AssertionError("the rounds did not settle")


def check(alg, data, cuts):
    want = P.trace(alg, oracle.encode(alg, data), data.size).copied.tolist()
    maps, carried = rounds(alg, data, cuts)
    assert maps[-1] == want, cuts
    agree = [next((k for k, (x, y) in enumerate(zip(m, want)) if x != y), len(want)) for m in maps]
    for k in range(len(maps) - 1):
        assert agree[k] == len(want) or agree[k + 1] >= agree[k] + 1, (k, agree)
    B = P.BS[alg]
    for ctx, m in carried:              # the in-order context under the map the words were published for
        _, before = block_sizes(alg, data, m)
        for r, c in enumerate(cuts[:-1]):
            b = c // B
            if b < len(before):
                assert ctx[r] == before[b], (r, c)
    return len(maps) - 1


def _text_with_bursts(n, seed):
    from density_b200 import synth
    d = synth.synth_text(n, first_page=seed).numpy().copy()
    for lo, ln in ((256 * 100 - 1024, 2048), (256 * 200, 1536), (256 * 300 - 512, 1024)):
        d[lo:lo + ln] = splitmix_bytes(ln, lo)
    return d


def _corpora():
    from density_b200 import synth
    dickens = np.fromfile(f"{GOLDEN_DIR}/dickens_200k.bin", dtype=np.uint8)[:96 * 1024 + 5]
    return {"noise": splitmix_bytes(40 * 1024 + 3, 3), "mixed": synth.synth_mixed(96 * 1024).numpy()[:96 * 1024 - 7],
            "bursts": _text_with_bursts(96 * 1024 + 1, 2), "dickens": dickens}


@pytest.mark.parametrize("alg", ["cheetah", "lion"])
@pytest.mark.parametrize("name", ["noise", "mixed", "bursts", "dickens"])
def test_rounds_settle_on_the_single_call_map(alg, name):
    data = _corpora()[name]
    n = data.size
    body = n // 256
    for cuts in ([0, 256 * 100, 256 * 201, n],                        # cuts that are not 16-block aligned for either block size
                 [0, 256 * 37, 256 * 37, 256 * (body - 3), n],         # an empty middle shard
                 [0, 0, 256 * 131, n]):                                # an empty first shard: the stream start on shard 1
        check(alg, data, [min(c, n) for c in cuts])
