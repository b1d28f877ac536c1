"""The single-device entries on an H100 (pytest -m gpu), at what they share: the argument rule of the stream-ordered entries, the buffer
kinds of the synchronous entries, and the diagnostics the context keeps.

- Refusals: encode_device / decode_device and their _path forms with d_out_size 4 bytes past an 8-byte boundary return
  DENSITY_B200_EARG and launch nothing; the same call with an aligned d_out_size then matches the oracle.
- Buffer kinds: every synchronous entry (an encode and a decode symbol per algorithm, decoded_size, chameleon_decode_range, and
  CodecInstance encode / decode on one reused instance) with the input pageable numpy, pinned torch, device, or device at an odd
  address, and the output likewise. Each gives the oracle's bytes and sizes, except that an encode refuses a device output at an odd
  address (encode_device's rule: the encoders store 2-byte words); pageable, pinned and aligned device buffers launch the same kernels.
- The diagnostic of the last run-parallel Cheetah decode survives a later call that grows the workspace, and density_b200_shutdown
  clears it until the next such decode."""
import ctypes

import numpy as np
import pytest

import oracle

pytestmark = pytest.mark.gpu
ALG_ID = {"chameleon": 0, "cheetah": 1, "lion": 2}
EARG = 4
MIB = 1 << 20
KINDS = ("pageable", "pinned", "device", "device_odd")


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
def text():
    from density_b200 import synth
    return synth.synth_text(MIB + 7).numpy()


@pytest.fixture(scope="module")
def streams(text):
    return {alg: oracle.encode(alg, text) for alg in ALG_ID}


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def buffer(torch, kind, data=None, n=None):
    """a buffer of `kind` holding `data`, or of n zero bytes"""
    a = np.zeros(n, np.uint8) if data is None else np.ascontiguousarray(data, np.uint8)
    if kind == "pageable":
        return a.copy()
    if kind == "pinned":
        return torch.from_numpy(a.copy()).pin_memory()
    off = 1 if kind == "device_odd" else 0
    buf = torch.zeros(a.size + off + 1, dtype=torch.uint8, device="cuda")
    buf[off:off + a.size] = torch.from_numpy(a.copy()).cuda()
    return buf[off:off + a.size]


def host(buf):
    return buf if isinstance(buf, np.ndarray) else buf.cpu().numpy()


# ---- refusals ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", list(ALG_ID))
@pytest.mark.parametrize("entry", ["encode_device", "decode_device", "encode_device_path", "decode_device_path"])
def test_misaligned_d_out_size_is_refused(torch_cuda, lib, text, streams, alg, entry):
    torch = torch_cuda
    encode = entry.startswith("encode")
    src = text if encode else streams[alg]
    want = streams[alg] if encode else text
    d_in = torch.from_numpy(src.copy()).cuda()
    cap = oracle.safe_encode_buffer_size(alg, text.size) if encode else text.size
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(4, dtype=torch.int64, device="cuda")
    fn = getattr(lib, f"density_b200_{entry}")

    def call(d_out_size):
        args = [ALG_ID[alg], d_in.data_ptr(), src.size, d_out.data_ptr(), cap, d_out_size, _stream(torch)]
        return fn(*(args + [0] if entry.endswith("_path") else args))

    torch.cuda.synchronize()
    before = lib.density_b200_kernel_launches()
    assert call(sizes.data_ptr() + 4) == EARG
    assert lib.density_b200_kernel_launches() == before, "a refused call launched kernels"
    assert call(sizes.data_ptr() + 8) == 0, lib.density_b200_last_error()
    torch.cuda.synchronize()
    n = int(sizes[1].item())
    assert n == want.size and (d_out[:n].cpu().numpy() == want).all()
    assert int(sizes[0].item()) == 0 and int(sizes[2].item()) == 0, "the refused call wrote its result"


# ---- the synchronous entries by buffer kind ---------------------------------------------------------------------------------------------
def _symbol(alg, encode):
    from density_b200 import CODECS
    C = CODECS[alg]
    return C.encode if encode else C.decode


def _cases(text, streams):
    """name -> (input, output size (None: no output), call(input, output) -> bytes written or size, expected bytes or size)"""
    from density_b200.codec import CODECS, Chameleon, CodecInstance
    cases = {}
    for alg in ALG_ID:
        cases[f"{alg}_encode"] = (text, oracle.safe_encode_buffer_size(alg, text.size), _symbol(alg, True), streams[alg])
        cases[f"{alg}_decode"] = (streams[alg], text.size, _symbol(alg, False), text)
        cases[f"{alg}_decoded_size"] = (streams[alg], None, lambda i, o, C=CODECS[alg]: C.decoded_size(i), text.size)
        inst = CodecInstance(alg)

        def inst_call(i, o, inst=inst, encode=True):
            inst.clear_state()
            return inst.encode(i, o) if encode else inst.decode(i, o)
        cases[f"{alg}_codec_encode"] = (text, oracle.safe_encode_buffer_size(alg, text.size), inst_call, streams[alg])
        cases[f"{alg}_codec_decode"] = (streams[alg], text.size, lambda i, o, f=inst_call: f(i, o, encode=False), text)
    first, length = 300001, 250003
    cases["chameleon_decode_range"] = (streams["chameleon"], length, lambda i, o: Chameleon.decode_range(i, first, o),
                                       text[first:first + length])
    return cases


CASES = [f"{a}_{op}" for a in ALG_ID for op in ("encode", "decode", "decoded_size", "codec_encode", "codec_decode")] + ["chameleon_decode_range"]


@pytest.mark.parametrize("case", CASES)
def test_sync_entries_by_buffer_kind(torch_cuda, lib, text, streams, case):
    from density_b200 import EncodeError
    torch = torch_cuda
    src, out_n, call, want = _cases(text, streams)[case]
    launches = {}
    for kin in KINDS:
        for kout in (KINDS if out_n is not None else ("none",)):
            what = f"{case}: input {kin}, output {kout}"
            i = buffer(torch, kin, src)
            o = buffer(torch, kout, n=out_n) if out_n is not None else None
            torch.cuda.synchronize()
            before = lib.density_b200_kernel_launches()
            if kout == "device_odd" and case.endswith("encode"):
                with pytest.raises(EncodeError):
                    call(i, o)
                continue
            r = call(i, o)
            if kin != "device_odd" and kout != "device_odd":
                launches[(kin, kout)] = lib.density_b200_kernel_launches() - before
            if o is None:
                assert r == want, what
                continue
            w = np.asarray(want, np.uint8)
            assert r == w.size, what
            got = host(o)[:r]
            assert (got == w).all(), f"{what}: first difference at {int(np.argmax(got != w))}"
    assert len(set(launches.values())) == 1, f"{case}: launch counts differ by buffer kind: {launches}"


# ---- the diagnostic of the last run-parallel Cheetah decode -----------------------------------------------------------------------------
def test_cheetah_decode_rounds_survive_workspace_growth(torch_cuda, lib, text, streams):
    from density_b200 import synth
    torch = torch_cuda
    big = synth.synth_text(64 * MIB, device="cuda")
    big_enc = torch.zeros(oracle.safe_encode_buffer_size("chameleon", big.numel()), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.density_b200_encode_device(0, big.data_ptr(), big.numel(), big_enc.data_ptr(), big_enc.numel(), sz.data_ptr(),
                                          _stream(torch)) == 0, lib.density_b200_last_error()
    torch.cuda.synchronize()
    big_n = int(sz.item())
    big_out = torch.zeros(big.numel(), dtype=torch.uint8, device="cuda")
    ch_in = torch.from_numpy(streams["cheetah"].copy()).cuda()
    ch_out = torch.zeros(text.size, dtype=torch.uint8, device="cuda")

    def cheetah_decode():
        assert lib.density_b200_decode_device_path(1, ch_in.data_ptr(), ch_in.numel(), ch_out.data_ptr(), ch_out.numel(), sz.data_ptr(),
                                                   _stream(torch), 0) == 0, lib.density_b200_last_error()
        torch.cuda.synchronize()
        assert int(sz.item()) == text.size

    def rounds():
        w = (ctypes.c_uint32 * 4)()
        return lib.density_b200_cheetah_decode_rounds(w), list(w)

    lib.density_b200_shutdown()                   # the workspace starts small, so the decode below has to grow it
    cheetah_decode()
    rc, first = rounds()
    assert rc == 0, lib.density_b200_last_error()
    assert lib.density_b200_decode_device(0, big_enc.data_ptr(), big_n, big_out.data_ptr(), big_out.numel(), sz.data_ptr(),
                                          _stream(torch)) == 0, lib.density_b200_last_error()
    torch.cuda.synchronize()
    assert int(sz.item()) == big.numel() and torch.equal(big_out, big)
    assert rounds() == (0, first), "the Cheetah decode diagnostic changed behind a Chameleon decode"
    lib.density_b200_shutdown()
    assert rounds()[0] == EARG
    assert lib.density_b200_decode_device(0, big_enc.data_ptr(), big_n, big_out.data_ptr(), big_out.numel(), sz.data_ptr(),
                                          _stream(torch)) == 0, lib.density_b200_last_error()
    torch.cuda.synchronize()
    assert rounds()[0] == EARG, "only a run-parallel Cheetah decode sets the diagnostic"
    cheetah_decode()
    assert rounds() == (0, first)
