"""The argument rule of the sharded decode pieces and drivers (include/density_b200.h; needs an H100: pytest -m gpu).

Every table, transfer, carry and word pointer is 4-byte aligned, d_out_size 8-byte and d_seam8 4-byte. A misaligned one returns
DENSITY_B200_EARG and enqueues nothing; the same piece then runs through its phases with aligned pointers and decodes to the bytes the
oracle encoded. The Lion piece and drivers have their own checks in test_gpu_sharded_lion_decode.py."""
import ctypes

import numpy as np
import pytest

import oracle

pytestmark = pytest.mark.gpu

EARG = 4


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


@pytest.fixture(scope="module")
def data():
    from density_b200 import synth
    return synth.synth_text(300 * 1024 + 5).numpy()    # no copy-mode block: the quiet Chameleon drivers decode it with verdict 0


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class Buffers:
    """one piece's device buffers: the stream, the output, a table, a carry, words, the size and the seam words"""

    def __init__(self, torch, alg, data):
        enc = oracle.encode(alg, data)
        self.n, self.cap = enc.size, data.size + 64
        self.d_in = torch.from_numpy(enc.copy()).cuda()
        self.d_out = torch.zeros(self.cap, dtype=torch.uint8, device="cuda")
        self.table = torch.zeros(3 * 65536 + 1, dtype=torch.int32, device="cuda")
        self.carry = torch.zeros(3 * 65536 + 1, dtype=torch.int32, device="cuda")
        self.words = torch.zeros(16, dtype=torch.int32, device="cuda")
        self.size = torch.zeros(2, dtype=torch.int64, device="cuda")
        self.seam = torch.zeros(9, dtype=torch.int32, device="cuda")
        self.flags = torch.ones(1, dtype=torch.int32, device="cuda")

    def decoded(self, torch, data):
        torch.cuda.synchronize()
        n = int(self.size[0].item())
        return n == data.size and bool((self.d_out[:n].cpu().numpy() == data).all())


def refused(lib, *calls):
    """every call returns DENSITY_B200_EARG and none of them enqueues a kernel"""
    before = lib.density_b200_kernel_launches()
    rcs = [c() for c in calls]
    assert rcs == [EARG] * len(calls)
    assert lib.density_b200_kernel_launches() == before


def test_cheetah_piece(torch_cuda, lib, data):
    torch, st = torch_cuda, _stream(torch_cuda)
    b = Buffers(torch, "cheetah", data)
    h = lib.density_b200_cheetah_decode_shard_create()
    ph1 = lambda t: lib.density_b200_cheetah_decode_shard_phase1(h, b.d_in.data_ptr(), b.n, b.d_out.data_ptr(), b.cap, 1, 1, t, st)
    ph2 = lambda c: lib.density_b200_cheetah_decode_shard_phase2(h, c, st)
    walk = lambda p, w: lib.density_b200_cheetah_decode_shard_round_walk(h, p, w, st)
    fold = lambda c, w: lib.density_b200_cheetah_decode_shard_round_fold(h, c, w, 1, 0, st)
    ph3 = lambda sz, seam: lib.density_b200_cheetah_decode_shard_phase3(h, sz, seam, st)
    t, c, w = b.table.data_ptr(), b.carry.data_ptr(), b.words.data_ptr()
    refused(lib, lambda: ph1(t + 2))                                               # d_cmap_out
    assert ph1(t) == 0
    refused(lib, lambda: ph2(c + 2))                                               # d_cmap_carry
    assert ph2(None) == 0
    for k in range(lib.density_b200_cheetah_decode_round_budget()):
        if k == 0:
            refused(lib, lambda: walk(t + 2, w), lambda: walk(t, w + 2))           # d_pred_out, d_words4
        assert walk(t, w) == 0
        if k == 0:
            refused(lib, lambda: fold(c + 2, w), lambda: fold(None, w + 2))       # d_pred_carry, d_all_words
        assert fold(None, w) == 0
    sz, seam = b.size.data_ptr(), b.seam.data_ptr()
    refused(lib, lambda: ph3(sz + 4, seam), lambda: ph3(sz, seam + 2))             # d_out_size, d_seam8
    assert ph3(sz, seam) == 0
    assert b.decoded(torch, data)
    lib.density_b200_cheetah_decode_shard_destroy(h)


def test_chameleon_piece(torch_cuda, lib, data):
    torch, st = torch_cuda, _stream(torch_cuda)
    b = Buffers(torch, "chameleon", data)
    h = lib.density_b200_decode_shard_create()
    t, c, sz, seam = b.table.data_ptr(), b.carry.data_ptr(), b.size.data_ptr(), b.seam.data_ptr()
    transfers = b.words.new_zeros(3200).data_ptr()

    def phase2(fn):                                                                # d_carry_in, d_out_size, d_seam8
        ph2 = lambda c, sz, seam: fn(h, c, b.d_out.data_ptr(), sz, seam, st)
        refused(lib, lambda: ph2(c + 2, sz, seam), lambda: ph2(None, sz + 4, seam), lambda: ph2(None, sz, seam + 2))
        b.size.zero_()
        assert ph2(None, sz, seam) == 0
        assert b.decoded(torch, data)
    ph1 = lambda t: lib.density_b200_decode_shard_phase1(h, b.d_in.data_ptr(), b.n, b.cap, 1, t, st)
    refused(lib, lambda: ph1(t + 2))                                               # d_table_out
    assert ph1(t) == 0
    phase2(lib.density_b200_decode_shard_phase2)
    assert lib.density_b200_decode_shard_prot_transfer(h, b.d_in.data_ptr(), b.n, b.cap, 1, transfers, st) == 0
    assert lib.density_b200_decode_shard_prot_phase1(h, transfers, 1, 0, t, st) == 0
    phase2(lib.density_b200_decode_shard_prot_phase2)
    lib.density_b200_decode_shard_destroy(h)


@pytest.mark.parametrize("alg", ["chameleon", "cheetah"])
def test_drivers(torch_cuda, lib, data, alg):
    torch, st = torch_cuda, _stream(torch_cuda)
    from density_b200 import sharded
    b = Buffers(torch, alg, data)
    dec = sharded.ShardedDecoder(torch.device("cuda"))
    d_in, d_out, fl = b.d_in.data_ptr(), b.d_out.data_ptr(), b.flags.data_ptr()
    if alg == "chameleon":
        known = (lib.density_b200_decode_sharded, lib.density_b200_decode_sharded_protected)
        stream = (lambda sz: lib.density_b200_decode_sharded_stream(dec._h, d_in, b.n, 0, d_out, b.cap, sz, None, fl, None, st),
                  lambda sz: lib.density_b200_decode_sharded_stream_protected(dec._h, d_in, b.n, 0, d_out, b.cap, sz, None, fl, None, st))
    else:
        known = (lib.density_b200_decode_sharded_cheetah, lib.density_b200_decode_sharded_cheetah_protected)
        stream = (lambda sz: lib.density_b200_decode_sharded_cheetah_stream(dec._h, d_in, b.n, 0, 0, d_out, b.cap, sz, None, fl, None, st),
                  lambda sz: lib.density_b200_decode_sharded_cheetah_stream_protected(dec._h, d_in, b.n, 0, d_out, b.cap, sz, None, fl, None, st))
    drivers = [lambda sz, fn=fn: fn(dec._h, d_in, b.n, d_out, b.cap, sz, fl, None, st) for fn in known] + list(stream)
    sz = b.size.data_ptr()
    refused(lib, *[lambda fn=fn: fn(sz + 4) for fn in drivers])                    # d_out_size
    for fn in drivers:
        b.size.zero_(); b.d_out.zero_(); b.flags.fill_(1)
        assert fn(sz) == 0, lib.density_b200_last_error()
        assert b.decoded(torch, data) and int(b.flags.item()) == 0
    dec.close()
