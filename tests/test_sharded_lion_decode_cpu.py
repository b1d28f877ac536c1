"""Sharded Lion decode on the CPU: the walk relayed from piece to piece, the protection transfers on the Lion geometry, and the kernels'
build for sm_90a.

- tests/lion_piece_model.cpp runs the row algorithm of lion_walk.cuh (the walk kernel's) over the pieces of oracle streams, each piece
  laid out in rows of its own and walked from the lists and last_hash the piece before it left; it must equal the walk of the whole
  stream at 1-9 cuts, empty pieces included.
- tests/prot_decode_model_lion.py models dec_prot_transfer<LionT>: composed from the stream start, the transfers must give the
  in-order automaton of the oracle's Lion stream (protection.trace) at every cut, with cuts inside copy runs and with a penalty pending
  at every counter phase.
- cl_decode.cu compiles for sm_90a and no kernel of the sharded Lion path spills."""
import ctypes
import functools
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import oracle
import prot_decode_model_lion as M
import protection as P
from conftest import payload

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ALG = "lion"
BS = P.BS[ALG]
MIB = 1 << 20


def _text(n, first_page=0):
    from density_b200 import synth
    return synth.synth_text(n, first_page=first_page).numpy()


# ---- the walk, piece by piece ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def piece_model(tmp_path_factory):
    so = os.path.join(str(tmp_path_factory.mktemp("lion_piece")), "lion_piece_model.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(HERE, "lion_piece_model.cpp"), "-o", so])
    L = ctypes.CDLL(so)
    L.lion_piece_model_check.restype = ctypes.c_long
    L.lion_piece_model_check.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)]
    return L


def walk_pieces(L, enc, cuts):
    enc = np.ascontiguousarray(enc, np.uint8)
    c = np.ascontiguousarray(cuts, np.uint64)
    counts = (ctypes.c_uint64 * 8)()
    nb = L.lion_piece_model_check(enc.ctypes.data, enc.size, c.ctypes.data, c.size, counts)
    return nb, list(counts)


@functools.lru_cache(maxsize=None)
def walk_corpora():
    from density_b200 import synth
    out = {"text": _text(MIB // 2 + 333, 3), "mixed": synth.synth_mixed(MIB // 2).numpy(), "zeros": np.zeros(200 * 1024 + 5, np.uint8),
           "dickens": np.fromfile(os.path.join(HERE, "golden", "dickens_200k.bin"), dtype=np.uint8)}
    return {k: oracle.encode(ALG, v) for k, v in out.items()}


@pytest.mark.parametrize("name", ["text", "mixed", "zeros", "dickens"])
def test_walk_piece_by_piece_equals_the_whole_walk(piece_model, name):
    enc = walk_corpora()[name]
    nb, _ = walk_pieces(piece_model, enc, [0, 1 << 40])
    assert nb > 100
    rng = np.random.default_rng(len(name))
    for k in range(1, 10):          # 1-9 cuts, odd block counts (rows split differently from the whole walk's) and empty pieces
        inner = sorted(int(v) for v in rng.integers(0, nb + 1, k))
        if k % 3 == 0:
            inner[k // 2] = inner[k // 2 - 1] if k > 1 else inner[0]
        cuts = [0] + inner + [nb]
        got, counts = walk_pieces(piece_model, enc, cuts)
        assert got == nb, (name, cuts)
        assert counts[0] == counts[4] and counts[1] == counts[5], counts


def test_walk_pieces_at_every_small_cut(piece_model):
    """one cut at each of the first 70 blocks, and a piece of one block at each of them, behind an empty piece"""
    enc = walk_corpora()["dickens"]
    nb, _ = walk_pieces(piece_model, enc, [0, 1 << 40])
    for b in range(70):
        assert walk_pieces(piece_model, enc, [0, b, nb])[0] == nb, b
        assert walk_pieces(piece_model, enc, [0, b, b, b + 1, nb])[0] == nb, b


# ---- the protection transfers on the Lion geometry ------------------------------------------------------------------------------------
def _bursts():
    data = _text(MIB // 2, first_page=5)
    rnd = payload("random", 64 * 1024, 7)
    cuts = [500 * 256, 1001 * 256, 1501 * 256]
    for i, c in enumerate(cuts):                    # a burst ending at the cut, one straddling it, one starting at it
        lo = [c - 2048, c - 1024, c][i]
        data[lo:lo + 2048] = rnd[i * 8192:i * 8192 + 2048]
    return data, [0] + cuts + [data.size]


@functools.lru_cache(maxsize=None)
def prot_corpora():
    from density_b200 import synth
    noise = payload("random", MIB // 4 + 77, 1)
    mixed = synth.synth_mixed(MIB // 2).numpy()
    out = [(noise, [0, 300 * 256, 700 * 256, noise.size]), (mixed, [0, 511 * 256, 1003 * 256, 1501 * 256, mixed.size]), _bursts()]
    res = []
    for data, cuts in out:
        enc = oracle.encode(ALG, data)
        res.append((data, cuts, enc, P.trace(ALG, enc, data.size)))
    return res


NAMES = ["noise", "synth_mixed", "text_bursts"]


def true_candidate(tr, b):
    return M.cand_index(*tr.state[b], tr.counter[b] % 16)


def _kind(tr, b):
    if tr.state[b][0] > 0 and not tr.copied[b - 1]:
        return "pending"
    return "run" if tr.copied[b] and tr.copied[b - 1] else None


def cut_blocks(tr, cuts):
    """the corpus' cuts plus, for every counter phase, a block with a penalty pending in front of it and one inside a copy run"""
    nb = len(tr.off)
    want = {c // BS for c in cuts[1:-1]}
    for ph in range(16):
        pend = [b for b in range(ph or 16, nb, 16) if _kind(tr, b) == "pending"]
        run = [b for b in range(ph or 16, nb, 16) if _kind(tr, b) == "run"]
        for kind in (pend, run):
            if kind:
                want.update({kind[0], kind[len(kind) // 2]})
    return [0] + sorted(b for b in want if 0 < b < nb) + [nb]


def offset(tr, b):
    return int(tr.off[b]) if b < len(tr.off) else tr.n_stream


def test_the_lion_geometry():
    assert (M.CH, M.BS, M.MAXBLK, M.NC) == (4096, 64, 70, 35) and P.CH[ALG] == 4096 and P.BS[ALG] == M.BS
    assert M.consumed_table(np.zeros(6, np.uint8))[0] == 6 + 16 * 4
    assert M.consumed_table(np.full(6, 255, np.uint8))[0] == 6 + 16 * 2          # flag 7 everywhere
    data = _text(64 * 1024, first_page=2)
    enc = oracle.encode(ALG, data)
    tr = P.trace(ALG, enc, data.size)
    cons = M.consumed_table(enc)
    full = [b for b in range(len(tr.off)) if not tr.copied[b] and (b + 1) * BS <= data.size]
    assert full and all(cons[tr.off[b]] == tr.size[b] for b in full)


@pytest.mark.parametrize("k", range(len(NAMES)), ids=NAMES)
def test_composed_transfers_are_the_in_order_automaton_at_every_cut(k):
    data, cuts, enc, tr = prot_corpora()[k]
    assert tr.copied.any()
    blocks = cut_blocks(tr, cuts)
    kinds = {(tr.counter[b] % 16, _kind(tr, b)) for b in blocks[1:-1]}
    if k < 2:          # noise and mixed data: a penalty pending and a copy run at a cut at every counter phase
        assert all((ph, kind) in kinds for ph in range(16) for kind in ("pending", "run")), sorted(kinds, key=str)
    transfers, max_live = [], 0
    for r, (a, b) in enumerate(zip(blocks[:-2], blocks[1:-1])):
        piece = enc[offset(tr, a):offset(tr, b)]
        T, stats = M.transfer(piece)
        transfers.append(T)
        max_live = max(max_live, stats["max_live"])
        x = M.compose(transfers, r + 1)
        assert x == true_candidate(tr, b), (r, b, x, tr.state[b], tr.counter[b])
        st = M.cand_state(M.compose(transfers, r))
        end = M.exact_walk(M.consumed_table(piece), piece.size, st)
        assert end is not None and end[1] == b - a and M.cand_index(*end[0]) == x
    assert max_live <= M.HEAD_CAP


def test_every_candidate_equals_its_own_in_order_walk():
    data, cuts, enc, tr = prot_corpora()[1]
    b0, b1 = cuts[1] // BS, cuts[2] // BS
    piece = enc[offset(tr, b0):offset(tr, b1)]
    T, _ = M.transfer(piece)
    cons = M.consumed_table(piece)
    rng = np.random.default_rng(3)
    for c in sorted({0, 1, 199, 200, 3199, true_candidate(tr, b0)} | set(rng.integers(0, M.NCAND, 80).tolist())):
        end = M.exact_walk(cons, piece.size, M.cand_state(c))
        want = M.NOEND if end is None else M.cand_index(*end[0])
        assert T[c] == want, (c, M.cand_state(c), T[c], want)


# ---- the build ---------------------------------------------------------------------------------------------------------------------------
NVCC = os.environ.get("NVCC") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc"))


@pytest.mark.skipif(not NVCC, reason="needs nvcc")
def test_the_sharded_lion_kernels_compile_for_sm90a_without_spills(tmp_path):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(ROOT, "density_b200", "csrc", "cl_decode.cu"), "-o", str(tmp_path / "cl_decode.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    props = {}
    cur = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            props[cur] = (int(m.group(1)), int(m.group(2)))
    wanted = {"cd_piece_endINS_6bounds5LionT": 0, "cd_piece_endINS_6bounds5CheeT": 0, "cd_seam_wordsILj64": 0, "7ld_walk": 0,
              "dec_prot_transferINS0_5LionTELb0": 0}
    for key in wanted:
        hits = [k for k in props if key in k]
        assert hits, (key, sorted(props))
        assert all(props[k] == (0, 0) for k in hits), {k: props[k] for k in hits}
    assert all(v == (0, 0) for v in props.values()), {k: v for k, v in props.items() if v != (0, 0)}
