"""Chameleon flag pass: the first quad of a tile is never the continuation of a run of equal quads (needs an H100: pytest -m gpu)."""
import numpy as np
import pytest

import oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device; there is no CPU fallback")
    return torch


@pytest.fixture(scope="module")
def codecs(torch_cuda):
    import density_b200
    density_b200.load()  # raises if the CUDA extension is missing
    return density_b200.CODECS


def test_chameleon_all_ones_record_at_tile_starts(torch_cuda, codecs):
    """Quad 0xEE4FF4DD has hash 0xFFFF and fingerprint 0xFFFF, so its flag-pass record word is 0xFFFFFFFF. As the first quad of a
    16 KiB tile it has no predecessor in the tile and must not be taken for the continuation of a run of equal quads: its first
    occurrence in bucket 0xFFFF (the stream's first quad) and its occurrences right after a different quad of that bucket are
    misses. Tile starts in many tiles of many runs; encode_device paths 0 and 1 and chameleon_encode."""
    torch = torch_cuda
    import density_b200
    from density_b200 import synth
    M, X = 0x9D6EF916, 0xEE4FF4DD
    assert ((X * M) & 0xFFFFFFFF) >> 16 == 0xFFFF and (((X * M) & 0xFFFE) | (X >> 31)) == 0xFFFF
    cand = np.random.default_rng(7).integers(0, 1 << 32, 1 << 22, dtype=np.uint64)
    Y = int(next(c for c in cand[(((cand * M) & 0xFFFFFFFF) >> 16) == 0xFFFF] if c != X))     # another quad of bucket 0xFFFF
    q = synth.synth_text(8 << 20).numpy().view(np.uint32).copy()
    q[0] = X                                          # first occurrence in the bucket
    for k in range(1, q.size // 4096):
        if k % 3 == 0:
            q[4096 * k - 1000] = Y                    # right after a different quad of the bucket
            q[4096 * k] = X
        elif k % 3 == 1:
            q[4096 * k] = X                           # right after itself: a hit
    data = q.view(np.uint8)
    want = oracle.encode("chameleon", data)
    for path in (0, 1):
        d_in = torch.from_numpy(data.copy()).cuda()
        d_out = torch.zeros(codecs["chameleon"].safe_encode_buffer_size(data.size) + 64, dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        density_b200.encode_device("chameleon", d_in, d_out, d_sz, path=path)
        torch.cuda.synchronize()
        n = int(d_sz.item())
        assert n == want.size and (d_out[:n].cpu().numpy() == want).all(), path
    out = np.zeros(codecs["chameleon"].safe_encode_buffer_size(data.size), dtype=np.uint8)
    m = codecs["chameleon"].encode(data, out)                                                 # chameleon_encode, host pointers
    assert m == want.size and (out[:m] == want).all()
