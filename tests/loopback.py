"""tests/loopback_nccl.cpp, the loopback collective library the multi-rank tests install in place of NCCL: its build and its ctypes
binding (the NCCL entry points, the test-only exports, the per-rank call log)."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

OK, INTERNAL, INVALID_USAGE = 0, 3, 5            # ncclResult_t
UINT8, UINT32 = 1, 3                             # ncclDataType_t
ALLGATHER, SEND, RECV = 1, 2, 3                  # ops of the call log


class UniqueId(ctypes.Structure):
    _fields_ = [("internal", ctypes.c_char * 128)]


def build(dirpath):
    """Compile tests/loopback_nccl.cpp into dirpath (a directory of this session's own) and load it. Returns (path, ctypes library)."""
    so = os.path.join(str(dirpath), "loopback_nccl.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(HERE, "loopback_nccl.cpp"), "-o", so])
    L = ctypes.CDLL(so)
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    sigs = {
        "ncclGetUniqueId": (ctypes.c_int, [ctypes.POINTER(UniqueId)]),
        "ncclCommInitRank": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.c_int, UniqueId, ctypes.c_int]),
        "ncclCommDestroy": (ctypes.c_int, [vp]),
        "ncclAllGather": (ctypes.c_int, [vp, vp, sz, ctypes.c_int, vp, vp]),
        "ncclSend": (ctypes.c_int, [vp, sz, ctypes.c_int, ctypes.c_int, vp, vp]),
        "ncclRecv": (ctypes.c_int, [vp, sz, ctypes.c_int, ctypes.c_int, vp, vp]),
        "ncclGroupStart": (ctypes.c_int, []),
        "ncclGroupEnd": (ctypes.c_int, []),
        "ncclGetErrorString": (ctypes.c_char_p, [ctypes.c_int]),
        "loopback_set_host_copy": (None, [ctypes.c_int]),
        "loopback_set_timeout_ms": (None, [ctypes.c_long]),
        "loopback_log_read": (ctypes.c_int, [ctypes.c_int, vp, ctypes.c_int]),
        "loopback_log_clear": (None, []),
    }
    for name, (res, args) in sigs.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    return so, L


def call_log(L, rank):
    """The call log of `rank`: [(op, count, datatype, peer)] in call order."""
    n = L.loopback_log_read(rank, None, 0)
    buf = np.zeros((max(n, 1), 4), np.int64)
    n = L.loopback_log_read(rank, buf.ctypes.data, n)
    return [tuple(int(v) for v in row) for row in buf[:n]]
