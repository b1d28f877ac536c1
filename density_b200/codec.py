"""Host-side mirror of the reference's codec interface for the accelerated path.

Mirrors `trait Codec` (/root/reference/src/codec/codec.rs:12-127) and the inherent associated functions of
Chameleon / Cheetah / Lion (/root/reference/src/algorithms/chameleon/chameleon.rs:39-53, cheetah.rs:47-65,
lion.rs:64-82): same names, same argument meaning (`encode(input, output) -> bytes written`), same sizing
contract (`safe_encode_buffer_size`). All work happens in libdensity_b200.so (CUDA, sm_90a).

Buffers may be: bytes / bytearray / memoryview / numpy uint8 arrays (host) or torch CUDA uint8 tensors
(device-resident, no staging copies).
"""
import ctypes

import numpy as np

from . import _lib

ALG_IDS = {"chameleon": 0, "cheetah": 1, "lion": 2}
_EMALFORMED = 3     # DENSITY_B200_EMALFORMED


class EncodeError(Exception):
    """/root/reference/src/errors/encode_error.rs:4-13"""


class DecodeError(Exception):
    """/root/reference/src/errors/decode_error.rs:4-13"""


def _ptr_len(buf, writable=False):
    """-> (address, nbytes, keepalive)"""
    try:
        import torch
        if isinstance(buf, torch.Tensor):
            if buf.dtype != torch.uint8 or not buf.is_contiguous():
                raise TypeError("torch buffers must be contiguous uint8")
            return buf.data_ptr(), buf.numel(), buf
    except ImportError:  # pragma: no cover
        pass
    if isinstance(buf, np.ndarray):
        if buf.dtype != np.uint8 or not buf.flags.c_contiguous:
            raise TypeError("numpy buffers must be contiguous uint8")
        if writable and not buf.flags.writeable:
            raise TypeError("output buffer is read-only")
        return buf.ctypes.data, buf.size, buf
    if isinstance(buf, (bytes, bytearray, memoryview)):
        if writable:
            if isinstance(buf, bytes):
                raise TypeError("output buffer must be writable (bytearray / numpy / torch)")
            a = np.frombuffer(buf, dtype=np.uint8)
        else:
            a = np.frombuffer(buf, dtype=np.uint8)
        return a.ctypes.data, a.size, a
    raise TypeError(f"unsupported buffer type {type(buf)!r}")


class _Codec:
    """One algorithm. The reference's instances own a dictionary (`state`); every public entry point used by its
    benches and FFI builds a fresh one per call (chameleon.rs:45-53), which is what this path accelerates."""
    NAME = None
    _BLOCK = None
    _UNIT = None
    _SIG = None

    @classmethod
    def block_size(cls):
        return cls._BLOCK

    @classmethod
    def decode_unit_size(cls):
        return cls._UNIT

    @classmethod
    def signature_significant_bytes(cls):
        return cls._SIG

    @classmethod
    def safe_encode_buffer_size(cls, size):
        """codec.rs:18-21 (computed by the library)."""
        return getattr(_lib.load(), f"{cls.NAME}_safe_encode_buffer_size")(size)

    @classmethod
    def encode(cls, input, output):
        """Encode `input` into `output`; returns the number of bytes written (codec.rs:72-80)."""
        ip, n, k1 = _ptr_len(input)
        op, cap, k2 = _ptr_len(output, writable=True)
        r = getattr(_lib.load(), f"{cls.NAME}_encode")(ip, n, op, cap)
        if r == 0 and n != 0:
            raise EncodeError(_lib.last_error() or "encode failed")
        return r

    @classmethod
    def decode(cls, input, output):
        """Decode `input` into `output`; returns the number of bytes written (codec.rs:82-126)."""
        ip, n, k1 = _ptr_len(input)
        op, cap, k2 = _ptr_len(output, writable=True)
        r = getattr(_lib.load(), f"{cls.NAME}_decode")(ip, n, op, cap)
        if r == 0 and n != 0:
            raise DecodeError(_lib.last_error() or "decode failed")
        return r

    @classmethod
    def decoded_size(cls, input):
        """The number of bytes `decode` writes for `input` (host buffer or torch CUDA tensor), found from the block boundaries without
        decoding. Raises DecodeError when the stream is malformed (decode would fail at any capacity)."""
        ip, n, k1 = _ptr_len(input)
        size = ctypes.c_uint64(0)
        rc = _lib.load().density_b200_decoded_size(ALG_IDS[cls.NAME], ip, n, ctypes.byref(size))
        if rc == _EMALFORMED:
            raise DecodeError(_lib.last_error() or "malformed stream")
        if rc != 0:
            raise _lib.DensityB200Error(f"density_b200_decoded_size rc={rc}: {_lib.last_error()}")
        return size.value

    # convenience: bytes in, bytes out
    @classmethod
    def encode_bytes(cls, data):
        a = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        out = np.empty(max(1, cls.safe_encode_buffer_size(a.size)), dtype=np.uint8)
        n = cls.encode(a, out)
        return out[:n].tobytes()

    @classmethod
    def decode_bytes(cls, data, original_size=None):
        """original_size None: the size comes from decoded_size (an extra pass over the block boundaries)."""
        a = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        if original_size is None:
            original_size = cls.decoded_size(a)
        out = np.empty(max(1, original_size), dtype=np.uint8)
        n = cls.decode(a, out)
        return out[:n].tobytes()


class Chameleon(_Codec):
    """chameleon.rs:138-147"""
    NAME, _BLOCK, _UNIT, _SIG = "chameleon", 256, 8, 8

    @classmethod
    def decode_range(cls, input, first, output, index=None):
        """Decode bytes [first, first + len(output)) of what `input` decodes to into `output`, without decoding the bytes in front of
        them; returns the number of bytes written, min(first + len(output), S) - first or 0 when first >= S (S: the decoded size).
        Host buffers or torch CUDA tensors of any alignment. Raises DecodeError when the stream is malformed. With `index` (what
        build_index returned for this stream) only the stream between the two checkpoints around the window is read and decoded; an
        index that does not describe the stream raises DensityB200Error, one whose stream decodes differently raises DecodeError."""
        ip, n, k1 = _ptr_len(input)
        op, cap, k2 = _ptr_len(output, writable=True)
        written = ctypes.c_uint64(0)
        if index is None:
            name = "density_b200_chameleon_decode_range"
            rc = _lib.load().density_b200_chameleon_decode_range(ip, n, first, op, cap, ctypes.byref(written))
        else:
            xp, xn, k3 = _ptr_len(index)
            name = "density_b200_chameleon_decode_range_indexed"
            rc = _lib.load().density_b200_chameleon_decode_range_indexed(ip, n, xp, xn, first, op, cap, ctypes.byref(written))
        if rc == _EMALFORMED:
            raise DecodeError(_lib.last_error() or "malformed stream")
        if rc != 0:
            raise _lib.DensityB200Error(f"{name} rc={rc}: {_lib.last_error()}")
        return written.value

    @classmethod
    def build_index(cls, input, interval=16 << 20):
        """The seek index of stream `input` (include/density_b200.h, "Chameleon seek index"): a checkpoint every `interval` decoded bytes
        (a positive multiple of 256). Returns bytes for a host input, a CUDA uint8 tensor for a CUDA tensor. Raises DecodeError when
        the stream is malformed."""
        ip, n, k1 = _ptr_len(input)
        L = _lib.load()
        bound = L.density_b200_chameleon_index_bytes(n, interval)
        if not bound:
            raise ValueError("interval must be a positive multiple of 256")
        try:
            import torch
            dev = isinstance(input, torch.Tensor) and input.is_cuda
        except ImportError:  # pragma: no cover
            dev = False
        out = torch.empty(bound, dtype=torch.uint8, device=input.device) if dev else np.empty(bound, dtype=np.uint8)
        op, _, k2 = _ptr_len(out, writable=True)
        size = ctypes.c_uint64(0)
        rc = L.density_b200_chameleon_index_build(ip, n, interval, op, bound, ctypes.byref(size))
        if rc == _EMALFORMED:
            raise DecodeError(_lib.last_error() or "malformed stream")
        if rc != 0:
            raise _lib.DensityB200Error(f"density_b200_chameleon_index_build rc={rc}: {_lib.last_error()}")
        return out[:size.value].clone() if dev else out[:size.value].tobytes()


class Cheetah(_Codec):
    """cheetah.rs:188-197"""
    NAME, _BLOCK, _UNIT, _SIG = "cheetah", 128, 4, 8


class Lion(_Codec):
    """lion.rs:317-326"""
    NAME, _BLOCK, _UNIT, _SIG = "lion", 64, 4, 6


CODECS = {"chameleon": Chameleon, "cheetah": Cheetah, "lion": Lion}


class CodecInstance:
    """A Codec instance that is reused across calls (`let mut c = Chameleon::new(); c.encode(a, ..); c.encode(b, ..)`,
    codec.rs:16,72,82): the dictionary survives until clear_state(); the protection state is fresh in every call."""

    def __init__(self, alg):
        self.alg = alg
        self._lib = _lib.load()
        self._h = self._lib.density_b200_codec_create(ALG_IDS[alg])
        if not self._h:
            raise _lib.DensityB200Error(_lib.last_error())

    def close(self):
        if getattr(self, "_h", None):
            self._lib.density_b200_codec_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def clear_state(self):
        if self._lib.density_b200_codec_clear_state(self._h):
            raise _lib.DensityB200Error(_lib.last_error())

    def encode(self, input, output):
        ip, n, k1 = _ptr_len(input)
        op, cap, k2 = _ptr_len(output, writable=True)
        r = self._lib.density_b200_codec_encode(self._h, ip, n, op, cap)
        if r == 0 and n != 0:
            raise EncodeError(_lib.last_error() or "encode failed")
        return r

    def decode(self, input, output):
        ip, n, k1 = _ptr_len(input)
        op, cap, k2 = _ptr_len(output, writable=True)
        r = self._lib.density_b200_codec_decode(self._h, ip, n, op, cap)
        if r == 0 and n != 0:
            raise DecodeError(_lib.last_error() or "decode failed")
        return r


# ---- stream-ordered device API (torch tensors) ------------------------------------------------------------------
def _stream_handle(stream):
    import torch
    s = torch.cuda.current_stream() if stream is None else stream
    return ctypes.c_void_p(s.cuda_stream)


def encode_device(alg, d_in, d_out, d_out_size, stream=None, path=0):
    """Enqueue an encode of CUDA uint8 tensor `d_in` into `d_out` on `stream` (default: torch's current stream).
    `d_out_size` is a CUDA int64/uint64 tensor with one element that receives the encoded size. No synchronisation."""
    L = _lib.load()
    rc = L.density_b200_encode_device_path(ALG_IDS[alg], d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), d_out.numel(),
                                           d_out_size.data_ptr(), _stream_handle(stream), path)
    if rc != 0:
        raise EncodeError(f"density_b200_encode_device rc={rc}: {_lib.last_error()}")


def decode_device(alg, d_in, n_in, d_out, d_out_size, stream=None, path=0):
    L = _lib.load()
    rc = L.density_b200_decode_device_path(ALG_IDS[alg], d_in.data_ptr(), n_in, d_out.data_ptr(), d_out.numel(),
                                           d_out_size.data_ptr(), _stream_handle(stream), path)
    if rc != 0:
        raise DecodeError(f"density_b200_decode_device rc={rc}: {_lib.last_error()}")


def decoded_size_device(alg, d_in, n_in, d_result, stream=None):
    """Enqueue the decoded-size query of the first `n_in` bytes of CUDA uint8 tensor `d_in` on `stream` (default: torch's current
    stream). `d_result` is a CUDA int64/uint64 tensor of two elements that receives {decoded size, verdict}, verdict 0 or 3
    (DENSITY_B200_EMALFORMED, size 0). No synchronisation."""
    L = _lib.load()
    rc = L.density_b200_decoded_size_device(ALG_IDS[alg], d_in.data_ptr(), n_in, d_result.data_ptr(), _stream_handle(stream))
    if rc != 0:
        raise DecodeError(f"density_b200_decoded_size_device rc={rc}: {_lib.last_error()}")


def decode_range_device(d_in, n_in, first, d_out, d_result, stream=None):
    """Enqueue the Chameleon range decode of bytes [first, first + d_out.numel()) of what the first `n_in` bytes of CUDA uint8 tensor
    `d_in` decode to, into CUDA uint8 tensor `d_out`, on `stream` (default: torch's current stream). `d_result` is a CUDA int64/uint64
    tensor of three elements that receives {bytes written, decoded size, verdict}, verdict 0 or 3 (DENSITY_B200_EMALFORMED). The call
    returns once the stream's earlier work and the block-boundary walk are done; the decode itself is left enqueued."""
    L = _lib.load()
    rc = L.density_b200_chameleon_decode_range_device(d_in.data_ptr(), n_in, first, d_out.numel(), d_out.data_ptr(), d_result.data_ptr(),
                                                        _stream_handle(stream))
    if rc != 0:
        raise DecodeError(f"density_b200_chameleon_decode_range_device rc={rc}: {_lib.last_error()}")


def index_build_device(d_in, n_in, interval, d_index, d_result, stream=None):
    """Enqueue the Chameleon seek index build of the first `n_in` bytes of CUDA uint8 tensor `d_in` into CUDA uint8 tensor `d_index`
    (at least density_b200_chameleon_index_bytes(n_in, interval) bytes), on `stream` (default: torch's current stream). `d_result` is a
    CUDA int64/uint64 tensor of three elements that receives {index bytes, decoded size, verdict}. The call returns once the stream's
    earlier work and the checkpoint walk are done; the snapshots are left enqueued. Raises DecodeError on a malformed stream (nothing is
    written to d_index then)."""
    L = _lib.load()
    rc = L.density_b200_chameleon_index_build_device(d_in.data_ptr(), n_in, interval, d_index.data_ptr(), d_index.numel(), d_result.data_ptr(),
                                                       _stream_handle(stream))
    if rc != 0:
        raise DecodeError(f"density_b200_chameleon_index_build_device rc={rc}: {_lib.last_error()}")


def decode_range_indexed_device(d_in, n_in, d_index, index_len, first, d_out, d_result, stream=None):
    """decode_range_device from the seek index in the first `index_len` bytes of CUDA uint8 tensor `d_index`: only the stream between the
    checkpoints around the window is decoded. The call returns once the index's directory has been read (one wait on `stream`), with
    the decode enqueued. Raises DecodeError when the index does not describe a stream of n_in bytes."""
    L = _lib.load()
    rc = L.density_b200_chameleon_decode_range_indexed_device(d_in.data_ptr(), n_in, d_index.data_ptr(), index_len, first, d_out.numel(),
                                                                d_out.data_ptr(), d_result.data_ptr(), _stream_handle(stream))
    if rc != 0:
        raise DecodeError(f"density_b200_chameleon_decode_range_indexed_device rc={rc}: {_lib.last_error()}")
