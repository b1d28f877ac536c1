"""The step order of the Chameleon and Cheetah decode pieces (include/density_b200.h; needs an H100: pytest -m gpu).

A locate, or a phase 1, ends whatever piece the shard held: the locate scratch is phase 1's workspace, and a new piece's phase 1 is
not the protected phase 1 its transfer was for. So after prot_transfer, a quiet locate, a protected locate or a quiet phase 1 leaves
nothing for prot_phase1 to continue: it returns DENSITY_B200_EARG and enqueues nothing. The same shard then runs the protected steps in
their order and decodes to the bytes the oracle encoded."""
import ctypes

import pytest

import oracle

pytestmark = pytest.mark.gpu

EARG = 4
LOCATE_MAP_WORDS = {"chameleon": 266, "cheetah": 142}                 # DENSITY_B200_[CHEETAH_]LOCATE_MAP_WORDS, u64
PROT_LOCATE_MAP_WORDS = {"chameleon": 422404, "cheetah": 217604}      # DENSITY_B200_[CHEETAH_]PROT_LOCATE_MAP_WORDS, u32


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
    return synth.synth_text(300 * 1024 + 5).numpy()


class Piece:
    """one whole stream as the only piece (world 1, rank 0) on a fresh shard of `alg`, and the calls of its steps"""

    def __init__(self, torch, lib, alg, data):
        self.torch, self.lib, self.alg, self.data = torch, lib, alg, data
        enc = oracle.encode(alg, data)
        self.n, self.cap = enc.size, data.size + 64
        self.st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.d_in = torch.from_numpy(enc.copy()).cuda()
        self.d_out = torch.zeros(self.cap, dtype=torch.uint8, device="cuda")
        self.table = torch.zeros(3 * 65536, dtype=torch.int32, device="cuda")
        self.transfer = torch.zeros(3200, dtype=torch.int32, device="cuda")
        self.words = torch.zeros(8, dtype=torch.int32, device="cuda")
        self.size = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.seam = torch.zeros(8, dtype=torch.int32, device="cuda")
        self.map = torch.zeros(LOCATE_MAP_WORDS[alg], dtype=torch.int64, device="cuda")
        self.pmap = torch.zeros(PROT_LOCATE_MAP_WORDS[alg], dtype=torch.int32, device="cuda")
        self.cham = alg == "chameleon"
        self.h = lib.density_b200_decode_shard_create() if self.cham else lib.density_b200_cheetah_decode_shard_create()
        assert self.h

    def close(self):
        (self.lib.density_b200_decode_shard_destroy if self.cham else self.lib.density_b200_cheetah_decode_shard_destroy)(self.h)

    def prot_transfer(self):
        L, a = self.lib, (self.h, self.d_in.data_ptr(), self.n)
        if self.cham:
            return L.density_b200_decode_shard_prot_transfer(*a, self.cap, 1, self.transfer.data_ptr(), self.st)
        return L.density_b200_cheetah_decode_shard_prot_transfer(*a, self.d_out.data_ptr(), self.cap, 1, 1, self.transfer.data_ptr(), self.st)

    def prot_phase1(self):
        fn = self.lib.density_b200_decode_shard_prot_phase1 if self.cham else self.lib.density_b200_cheetah_decode_shard_prot_phase1
        return fn(self.h, self.transfer.data_ptr(), 1, 0, self.table.data_ptr(), self.st)

    def locate(self):
        L, a = self.lib, (self.h, self.d_in.data_ptr(), self.n, 0)
        if self.cham:
            return L.density_b200_decode_locate(*a, self.map.data_ptr(), self.st)
        return L.density_b200_cheetah_decode_locate(*a, 0, self.map.data_ptr(), self.st)

    def prot_locate(self):
        fn = self.lib.density_b200_decode_prot_locate if self.cham else self.lib.density_b200_cheetah_decode_prot_locate
        return fn(self.h, self.d_in.data_ptr(), self.n, 0, self.pmap.data_ptr(), self.st)

    def phase1(self):
        L, a = self.lib, (self.h, self.d_in.data_ptr(), self.n)
        if self.cham:
            return L.density_b200_decode_shard_phase1(*a, self.cap, 1, self.table.data_ptr(), self.st)
        return L.density_b200_cheetah_decode_shard_phase1(*a, self.d_out.data_ptr(), self.cap, 1, 1, self.table.data_ptr(), self.st)

    def decode_protected(self):
        """prot_transfer -> prot_phase1 -> the rest of the piece; True when it decodes to the original bytes"""
        L, T = self.lib, self.torch
        self.size.zero_(); self.d_out.zero_()
        assert self.prot_transfer() == 0, L.density_b200_last_error()
        assert self.prot_phase1() == 0, L.density_b200_last_error()
        sz, seam = self.size.data_ptr(), self.seam.data_ptr()
        if self.cham:
            assert L.density_b200_decode_shard_prot_phase2(self.h, None, self.d_out.data_ptr(), sz, seam, self.st) == 0
        else:
            assert L.density_b200_cheetah_decode_shard_phase2(self.h, None, self.st) == 0
            for _ in range(L.density_b200_cheetah_decode_round_budget()):
                assert L.density_b200_cheetah_decode_shard_round_walk(self.h, None, self.words.data_ptr(), self.st) == 0
                assert L.density_b200_cheetah_decode_shard_round_fold(self.h, None, self.words.data_ptr(), 1, 0, self.st) == 0
            assert L.density_b200_cheetah_decode_shard_phase3(self.h, sz, seam, self.st) == 0
        T.cuda.synchronize()
        m = int(self.size.item())
        return m == self.data.size and bool((self.d_out[:m].cpu().numpy() == self.data).all()) and int(self.seam[2].item()) == 0


@pytest.mark.parametrize("alg", ["chameleon", "cheetah"])
@pytest.mark.parametrize("between", ["locate", "prot_locate", "phase1"])
def test_prot_phase1_after_a_new_piece_is_refused(torch_cuda, lib, data, alg, between):
    p = Piece(torch_cuda, lib, alg, data)
    try:
        assert p.prot_transfer() == 0, lib.density_b200_last_error()
        assert getattr(p, between)() == 0, lib.density_b200_last_error()
        before = lib.density_b200_kernel_launches()
        assert p.prot_phase1() == EARG
        assert lib.density_b200_kernel_launches() == before
        assert p.decode_protected()
    finally:
        torch_cuda.cuda.synchronize()
        p.close()
