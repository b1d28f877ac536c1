"""Multi-GPU sharding of ONE bit-exact Chameleon stream (SURVEY.md §8e): one process per GPU, torch.distributed for the
only exchange step the path has — the 256 KiB last-writer tables.

Rank r owns bytes [r*S, (r+1)*S) of the stream (S a multiple of 256 so block grids line up).
  phase 1 (local)   flag pass with unknown carry-in; exports the shard's last-writer table   (density_b200_shard_phase1)
  exchange          all_gather of the tables (world * 256 KiB), left fold of ranks < r        (this file)
  phase 2 (local)   resolve first touches against the carried-in dictionary, scan, emit       (density_b200_shard_phase2)
The concatenation of the per-rank outputs is byte-identical to one chameleon_encode call over the whole buffer as long as
the protection automaton stays quiet (flags bit 0 reports otherwise). Outputs stay where they were produced; a caller
that wants them on one rank gathers them with the sizes returned here.

Input on which the protection automaton fires (copy mode) goes through ShardedChameleonEncoder.encode_protected or
ShardedEncoder.encode_protected instead: the copy-map iteration runs over all ranks, every round exchanging the tables, each rank's
automaton transfer (compose_prot_transfers is its numpy twin) and 4 round words, for a fixed budget of rounds.

Decode is the mirror image: rank r decodes its piece back into its shard with the same table exchange and fold. The decode
phase 1 (boundaries, writer pass) needs no carry-in and exports the piece's table; phase 2 decodes from the folded carry-in
and writes 8 seam words, which every rank gathers and judges with `seam_verdict`. Pieces with copy-mode blocks decode through
ShardedChameleonDecoder.decode_protected or ShardedDecoder.decode_protected: every piece first exports its protection transfer
(where its boundary walk ends for every automaton state and counter phase it may be entered in; compose_decode_prot_transfers is
the numpy twin of the composition), and phase 1 starts from the composed state.

Cheetah and Lion shard the same way with three phases around two exchanges (ShardedCLEncoder): the last quad of every shard (the
context of the next shard's first quad), then the shard's prediction transfer (P table), then its chunk-map transfer (C table). A
transfer says what the shard does to the state carried into it; the carry-in of rank r is the stream-start state folded with the
transfers of ranks < r (density_b200_cl_table_init / _fold, on the device). Only rank 0 may use copy mode; the seam verdict refuses
what would need it elsewhere. ShardedCLEncoder.encode_protected and ShardedEncoder.encode_protected(..., alg="cheetah" / "lion")
accept copy mode anywhere: the shard at the stream start settles its own map first, then every round runs the three phases on all
ranks and exchanges the automaton transfers and 8 round words (which carry each shard's last encoded quad), as Chameleon does.

A sharded Cheetah stream decodes the same way in pieces (ShardedDecoder.decode(..., alg="cheetah"), or the piece phases
density_b200_cheetah_decode_shard_* with fold_cheetah_cmap and fold_cl_tables for the exchanges): the chunk-map transfers are
exchanged once, then every prediction round exchanges each piece's prediction transfer and 4 round words, for a fixed budget of rounds.
Pieces with copy-mode blocks (ShardedDecoder.decode_protected(..., alg="cheetah"), or density_b200_cheetah_decode_shard_prot_transfer and
_prot_phase1 in place of phase 1) first exchange their protection transfers, as Chameleon's do.

A sharded Lion stream decodes in pieces too (ShardedLionDecoder, or the piece phases density_b200_lion_decode_shard_* with
fold_cheetah_cmap for the one exchange of chunk-map transfers). Lion has no prediction rounds: each piece's walk starts from the
prediction lists and context the piece before it left, so the walk's state (DENSITY_B200_LION_STATE_WORDS u32, 1.25 MiB) is relayed
from rank to rank and the pieces walk one after the other. Pieces with copy-mode blocks (ShardedLionDecoder.decode_protected) first
exchange their protection transfers, as Cheetah's do.

A stream whose cuts are not known (one chameleon_encode call, the reference library, a file) is cut at byte ranges instead
(`stream_ranges`): rank r holds its range and a halo of the next 264 bytes, computes the range map of every possible entry offset
(density_b200_decode_locate), and after an all_gather of the maps `locate_piece` gives every rank the exact offset where its
first block starts. The located piece then decodes as above.

A Cheetah stream without known cuts takes the same layout (ShardedDecoder.decode_stream(..., alg="cheetah", range_offset=o_r), or
density_b200_cheetah_decode_locate with `locate_piece(maps, rank, alg="cheetah")` and the piece phases). Its stream start has
copy-mode blocks, so the range that holds it (range_offset 0) finds its exit with the exact boundary walk; every later range uses
its candidate rows.
"""
import ctypes

import numpy as np
import torch
import torch.distributed as dist

from . import _lib

TABLE_ENTRIES = 65536
TOUCHED = 0x10000


def _rank_world(group=None):
    """(rank, world) of this process in `group`; (0, 1) without torch.distributed"""
    if not dist.is_initialized():
        return 0, 1
    return dist.get_rank(group), dist.get_world_size(group)


def _stream():
    """torch's current CUDA stream, as the library takes it"""
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, what):
    if rc:
        raise _lib.DensityB200Error(f"{what} rc={rc}: {_lib.last_error()}")


def gather_rows(t, group=None):
    """all_gather of every rank's `t`: [world, t.numel()] in rank order (world 1: a view of t)"""
    world = _rank_world(group)[1]
    if world == 1:
        return t.view(1, -1)
    out = torch.empty((world, t.numel()), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out.view(-1), t.contiguous(), group=group)
    return out


def initial_table(device):
    """Dictionary state at the stream start: only bucket 0 'holds quad 0' (chameleon.rs:41,89-91)."""
    t = torch.zeros(TABLE_ENTRIES, dtype=torch.int32, device=device)
    t[0] = TOUCHED
    return t


def fold_tables(gathered, rank):
    """carry-in of `rank` = left fold of the tables of ranks < rank over the initial state.
    gathered: int32 [world, 65536] (bit 16 = touched, low 16 bits = fingerprint). Pure tensor ops: runs on CPU (gloo
    tests) and CUDA alike."""
    carry = initial_table(gathered.device)
    for r in range(rank):
        t = gathered[r]
        carry = torch.where((t & TOUCHED) != 0, t, carry)
    return carry


SEAM_WORDS = 8


def seam_verdict(words):
    """The Python twin of cham_seam_verdict_k. words: int32 [world, 8], one row per piece in stream order:
    {first block incompressible, last block incompressible, not quiet or error, has blocks, size lo, size hi, 0, 0}.
    Returns (flags, total, offsets): flags 1 when a piece is not quiet or a seam joins two incompressible blocks (the
    protection automaton would fire across the cut, protection_state.rs:38-43), else 0; total = the summed sizes;
    offsets = int64 [world + 1], the prefix sums of the sizes. Pieces without blocks are skipped at the seams."""
    w = words.to("cpu", torch.int64) & 0xFFFFFFFF
    sizes = w[:, 4] | (w[:, 5] << 32)
    offsets = torch.zeros(w.shape[0] + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(sizes, 0)
    bad, prev_inc = bool((w[:, 2] != 0).any()), False
    for r in range(w.shape[0]):
        if w[r, 3]:
            bad |= prev_inc and bool(w[r, 0])
            prev_inc = bool(w[r, 1])
    return int(bad), int(offsets[-1]), offsets


PROT_TRANSFER_WORDS = 200  # DENSITY_B200_PROT_TRANSFER_WORDS: candidate states of the protection automaton
PROT_ROUND_WORDS = 4       # DENSITY_B200_PROT_ROUND_WORDS
CL_PROT_ROUND_WORDS = 8    # DENSITY_B200_CL_PROT_ROUND_WORDS: the round words of the Cheetah / Lion path, quad words at 4-5
PROT_STATUS_WORDS = 20     # DENSITY_B200_PROT_STATUS_WORDS
PROT_ESC = 0xFFFF          # a path that left the candidate states
_PC_NS, _PC_NP = 10, 10    # candidate starts 1..10, penalties 0..9 (chameleon_encode.cu: PC_NS, PC_NP)


def prot_candidate(state):
    """(penalty, start, previous_incompressible) -> the candidate index of a transfer entry (pc_encode), PROT_ESC outside the set."""
    p, s, prev = state
    if p >= _PC_NP or s < 1 or s > _PC_NS:
        return PROT_ESC
    return (int(prev) * _PC_NS + (s - 1)) * _PC_NP + p


def prot_state(c):
    """The inverse of prot_candidate (pc_decode); None for PROT_ESC."""
    if c == PROT_ESC:
        return None
    return (c % _PC_NP, (c // _PC_NP) % _PC_NS + 1, c // (_PC_NP * _PC_NS))


def compose_prot_transfers(transfers, rank):
    """The numpy twin of cham_prot_enter_k's composition: the candidate state entering shard `rank`, the transfers of shards < rank
    (int [world, PROT_TRANSFER_WORDS], entry c = candidate at the shard end when entered in candidate c, or PROT_ESC) applied in order
    to the stream-start state (candidate 0). PROT_ESC once a path leaves the candidates."""
    t = np.asarray(transfers).astype(np.int64) & 0xFFFFFFFF
    x = 0
    for r in range(rank):
        if x == PROT_ESC:
            break
        x = int(t[r, x])
    return x


DECODE_PROT_TRANSFER_WORDS = 3200   # DENSITY_B200_DECODE_PROT_TRANSFER_WORDS: (candidate state, counter mod 16) of a decode
DECODE_PROT_NOEND = 0xFFFE          # a decode transfer entry whose boundary walk does not end on the cut


def decode_prot_candidate(state, phase):
    """(penalty, start, previous_incompressible), counter mod 16 -> the candidate index of a decode transfer entry, PROT_ESC outside
    the set"""
    c = prot_candidate(state)
    return PROT_ESC if c == PROT_ESC else phase * PROT_TRANSFER_WORDS + c


def compose_decode_prot_transfers(transfers, rank):
    """The numpy twin of dec_prot_enter_k: the decode candidate entering piece `rank`, the transfers of pieces < rank (int [world,
    DECODE_PROT_TRANSFER_WORDS], entry c = candidate at the piece end when entered in candidate c, PROT_ESC or DECODE_PROT_NOEND)
    applied in order to the stream start (candidate 0). The first PROT_ESC / DECODE_PROT_NOEND met is returned: the pieces are
    refused."""
    t = np.asarray(transfers).astype(np.int64) & 0xFFFFFFFF
    x = 0
    for r in range(rank):
        if x >= DECODE_PROT_TRANSFER_WORDS:
            break
        x = int(t[r, x])
    return x


LOCATE_MAP_WORDS = 266     # DENSITY_B200_LOCATE_MAP_WORDS
CHEETAH_LOCATE_MAP_WORDS = 142   # DENSITY_B200_CHEETAH_LOCATE_MAP_WORDS
CHUNK = 16384              # non-last ranges are multiples of the boundary walk's chunk
HALO = 264                 # the largest Chameleon block: every byte a block starting inside a range can reach


def stream_ranges(total, world):
    """[(offset, n_range, n_halo)] per rank for a stream of `total` bytes: equal ranges rounded down to 16 KiB, the last rank takes
    the rest; each halo is the next min(264, bytes after the range) stream bytes."""
    per = total // world // CHUNK * CHUNK
    out = []
    for r in range(world):
        off = r * per
        n = per if r < world - 1 else total - off
        out.append((off, n, min(HALO, total - off - n)))
    return out


def locate_piece(maps, rank, alg="chameleon"):
    """density_b200_locate_piece (host only) on the gathered range maps, uint64-compatible [world, 266] in rank order. Returns
    (start, end, blocks_before, is_final): this rank's piece is its buffer's bytes [start, end). alg "cheetah": the Cheetah maps
    [world, 142] (density_b200_cheetah_locate_piece), and the tuple ends with is_first (the piece holds the stream start)."""
    cheetah = _alg_id(alg) == 1
    words, nout = (CHEETAH_LOCATE_MAP_WORDS, 5) if cheetah else (LOCATE_MAP_WORDS, 4)
    m = np.ascontiguousarray(np.asarray(maps).astype(np.uint64, copy=False).reshape(-1, words))
    out = (ctypes.c_uint64 * nout)()
    lib = _lib.load()
    fn = lib.density_b200_cheetah_locate_piece if cheetah else lib.density_b200_locate_piece
    _check(fn(m.ctypes.data, m.shape[0], rank, out), "locate_piece")
    return tuple(int(v) for v in out)


PROT_LOCATE_MAP_WORDS = 422404           # DENSITY_B200_PROT_LOCATE_MAP_WORDS: 4 header words + 132 entries x 3200 candidates
CHEETAH_PROT_LOCATE_MAP_WORDS = 217604   # DENSITY_B200_CHEETAH_PROT_LOCATE_MAP_WORDS: 4 + 68 x 3200


def prot_locate_piece(maps, rank, alg="chameleon"):
    """density_b200_prot_locate_piece (host only) on the gathered protected range maps, uint32-compatible [world, map words] in rank
    order. Returns (start, end, is_final, is_first, entry candidate, refused): this rank's piece is its buffer's bytes [start, end),
    entered in that decode candidate; refused != 0 on every rank when the composition met 0xFFFF / 0xFFFE anywhere."""
    alg = _alg_id(alg)
    if alg not in (0, 1):
        raise ValueError("prot_locate_piece: alg must be 'chameleon' or 'cheetah'")
    words = CHEETAH_PROT_LOCATE_MAP_WORDS if alg == 1 else PROT_LOCATE_MAP_WORDS
    m = np.ascontiguousarray(np.asarray(maps).astype(np.uint32, copy=False).reshape(-1, words))
    out = (ctypes.c_uint64 * 6)()
    _check(_lib.load().density_b200_prot_locate_piece(alg, m.ctypes.data, m.shape[0], rank, out), "prot_locate_piece")
    return tuple(int(v) for v in out)


class _Handle:
    """Owns one library handle: made by `create`, freed by `destroy` on close() or when the object is collected."""

    def _open(self, create, destroy, *args):
        self._lib = _lib.load()
        self._destroy = getattr(self._lib, destroy)
        self._h = getattr(self._lib, create)(*args)
        if not self._h:
            raise _lib.DensityB200Error(_lib.last_error())

    def close(self):
        if getattr(self, "_h", None):
            self._destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ShardedChameleonEncoder(_Handle):
    def __init__(self):
        self._open("density_b200_shard_create", "density_b200_shard_destroy")

    def encode_protected(self, d_in, d_out, d_size, group=None):
        """The copy-mode path (density_b200_shard_prot_*): d_in / d_out / d_size as in encode, any input. Runs the round budget of the
        copy-map iteration with torch.distributed exchanges (tables, transfers, round words) and the device folds. Returns
        seam_verdict's (flags, total, offsets) over all ranks; flags != 0 only when the map did not settle, the automaton left the
        candidate states, or on an error: the pieces are then void."""
        rank, world = _rank_world(group)
        stream = _stream()
        dev = d_in.device
        lib = self._lib

        def check(rc, what):
            _check(rc, f"shard_prot_{what}")

        n = d_in.numel()
        first_block = int(gather_rows(torch.tensor([n], dtype=torch.int64, device=dev), group)[:rank].sum()) // 256
        table = torch.empty(TABLE_ENTRIES, dtype=torch.int32, device=dev)
        transfer = torch.empty(PROT_TRANSFER_WORDS, dtype=torch.int32, device=dev)
        words = torch.empty(PROT_ROUND_WORDS, dtype=torch.int32, device=dev)
        check(lib.density_b200_shard_prot_phase1(self._h, d_in.data_ptr(), n, first_block, int(rank == world - 1), table.data_ptr(),
                                                 stream), "phase1")
        all_words = None
        for k in range(lib.density_b200_prot_round_budget()):
            if k:
                check(lib.density_b200_shard_prot_next(self._h, all_words.data_ptr(), world, table.data_ptr(), stream), "next")
            carry = fold_tables(gather_rows(table, group), rank).contiguous()
            check(lib.density_b200_shard_prot_transfer(self._h, carry.data_ptr(), transfer.data_ptr(), stream), "transfer")
            all_transfers = gather_rows(transfer, group).contiguous()
            check(lib.density_b200_shard_prot_settle(self._h, all_transfers.data_ptr(), world, rank, words.data_ptr(), stream), "settle")
            all_words = gather_rows(words, group).contiguous()
        check(lib.density_b200_shard_prot_next(self._h, all_words.data_ptr(), world, None, stream), "next")
        seam = torch.empty(SEAM_WORDS, dtype=torch.int32, device=dev)
        check(lib.density_b200_shard_prot_finish(self._h, d_out.data_ptr(), d_out.numel(), d_size.data_ptr(), seam.data_ptr(), stream),
              "finish")
        return seam_verdict(gather_rows(seam, group))

    def prot_status(self):
        """density_b200_shard_prot_status after encode_protected (waits for the device): dict with rounds (until settled, 0: not
        settled), settled, in_state ((penalty, start, previous_incompressible) entering the shard, None: left the candidates), esc and
        changed (this shard's blocks whose copy status changed, per round, 16 values)."""
        out = (ctypes.c_uint32 * PROT_STATUS_WORDS)()
        _check(self._lib.density_b200_shard_prot_status(self._h, out), "shard_prot_status")
        v = list(out)
        ins = None if v[2] == 0xFFFFFFFF else (v[2] & 0xFF, (v[2] >> 8) & 0xFF, v[2] >> 16)
        return {"rounds": v[0], "settled": v[1], "in_state": ins, "esc": v[3], "changed": v[4:20]}

    def encode(self, d_in, d_out, d_size, d_flags, group=None):
        """d_in / d_out: CUDA uint8 tensors (this rank's shard / its output buffer); d_size: int64[1]; d_flags: int32[1].
        Everything is enqueued on torch's current stream; the all_gather is the only collective."""
        rank, world = _rank_world(group)
        stream = _stream()
        table = torch.empty(TABLE_ENTRIES, dtype=torch.int32, device=d_in.device)
        _check(self._lib.density_b200_shard_phase1(self._h, d_in.data_ptr(), d_in.numel(), int(rank == world - 1), table.data_ptr(), stream),
               "shard_phase1")
        gathered = gather_rows(table, group)
        carry_ptr = None
        if rank > 0:
            self._carry = fold_tables(gathered, rank)
            carry_ptr = self._carry.data_ptr()
        _check(self._lib.density_b200_shard_phase2(self._h, carry_ptr, d_out.data_ptr(), d_out.numel(), d_size.data_ptr(), d_flags.data_ptr(),
                                                   stream), "shard_phase2")


ALGS = {"chameleon": 0, "cheetah": 1, "lion": 2}
CL_TABLE_P, CL_TABLE_C = 0, 1


def _alg_id(alg):
    return ALGS[alg] if isinstance(alg, str) else int(alg)


def _fold_on_device(gathered, rank, init, fold, what):
    """carry-in of `rank`: the stream-start state (init) folded with the rows of ranks < rank in order (fold), enqueued on torch's
    current stream. gathered: CUDA int32 [world, words]."""
    stream = _stream()
    carry = torch.empty(gathered.shape[1], dtype=torch.int32, device=gathered.device)
    rc = init(carry.data_ptr(), stream)
    for r in range(rank):
        if rc == 0:
            rc = fold(carry.data_ptr(), gathered[r].contiguous().data_ptr(), stream)
    _check(rc, what)
    return carry


def fold_cl_tables(alg, kind, gathered, rank):
    """carry-in of `rank` for the Cheetah / Lion sharded encode: the stream-start state (density_b200_cl_table_init) folded with the
    tables of ranks < rank in order (density_b200_cl_table_fold). gathered: CUDA int32 [world, words]. Enqueued on torch's current
    stream."""
    lib = _lib.load()
    alg = _alg_id(alg)
    return _fold_on_device(gathered, rank, lambda acc, st: lib.density_b200_cl_table_init(alg, kind, acc, st),
                           lambda acc, nxt, st: lib.density_b200_cl_table_fold(alg, kind, acc, nxt, st), "cl_table_init / fold")


def fold_cheetah_cmap(gathered, rank):
    """carry-in of piece `rank` for the sharded Cheetah decode: the stream-start chunk map (density_b200_cheetah_cmap_init) folded with
    the chunk-map transfers of pieces < rank in order (density_b200_cheetah_cmap_fold). gathered: CUDA int32 [world, 3 * 65536].
    Enqueued on torch's current stream."""
    lib = _lib.load()
    return _fold_on_device(gathered, rank, lib.density_b200_cheetah_cmap_init, lib.density_b200_cheetah_cmap_fold,
                           "cheetah_cmap_init / fold")


class ShardedCLEncoder(_Handle):
    """Sharded Cheetah / Lion encode through the shard phases, with torch.distributed for the exchanges (the phase-level twin of
    ShardedEncoder.encode(..., alg=...)). Rank r's d_in is bytes [o_r, o_r + n_r) of one input; non-final shards are multiples of 256
    bytes. The concatenation of the pieces equals one cheetah_encode / lion_encode call over the whole input when flags == 0."""

    def __init__(self, alg):
        self.alg = _alg_id(alg)
        self._open("density_b200_cl_shard_create", "density_b200_cl_shard_destroy", self.alg)
        self.words_p = self._lib.density_b200_cl_table_words(self.alg, CL_TABLE_P)
        self.words_c = self._lib.density_b200_cl_table_words(self.alg, CL_TABLE_C)
        self.events = None

    def encode(self, d_in, d_out, d_size, group=None, timing=False):
        """d_in: CUDA uint8 tensor (4-byte aligned), this rank's shard; d_out: its output buffer (2-byte aligned); d_size: int64[1].
        Returns seam_verdict's (flags, total, offsets) over all ranks; flags != 0: the pieces are void and the caller encodes on one
        device. timing: record CUDA events around the phases in self.events (phase 1, P exchange + fold, phase 2, C exchange + fold,
        phase 3 + seams)."""
        rank, world = _rank_world(group)
        stream = _stream()
        dev = d_in.device
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)] if timing else None
        mark = (lambda k: ev[k].record()) if timing else (lambda k: None)
        n = d_in.numel()
        last = torch.zeros(2, dtype=torch.int32, device=dev)        # {has a quad, last quad}: the next shard's first context
        if n >= 4:
            last[0] = 1
            last[1:] = d_in[n // 4 * 4 - 4:n // 4 * 4].clone().view(torch.int32)
        quads = gather_rows(last, group)
        prev = None
        if rank > 0:
            prev = torch.zeros(1, dtype=torch.int32, device=dev)
            for r in range(rank):
                prev = torch.where(quads[r, 0] != 0, quads[r, 1:2], prev)
        mark(0)
        tp = torch.empty(self.words_p, dtype=torch.int32, device=dev)
        _check(self._lib.density_b200_cl_shard_phase1(self._h, d_in.data_ptr(), n, int(rank == world - 1),
                                                      prev.data_ptr() if prev is not None else None, tp.data_ptr(), stream), "cl_shard_phase1")
        mark(1)
        carry_p = fold_cl_tables(self.alg, CL_TABLE_P, gather_rows(tp, group), rank) if rank > 0 else None
        mark(2)
        tc = torch.empty(self.words_c, dtype=torch.int32, device=dev)
        _check(self._lib.density_b200_cl_shard_phase2(self._h, carry_p.data_ptr() if carry_p is not None else None, tc.data_ptr(), stream),
               "cl_shard_phase2")
        mark(3)
        carry_c = fold_cl_tables(self.alg, CL_TABLE_C, gather_rows(tc, group), rank) if rank > 0 else None
        mark(4)
        words = torch.empty(SEAM_WORDS, dtype=torch.int32, device=dev)
        _check(self._lib.density_b200_cl_shard_phase3(self._h, carry_c.data_ptr() if carry_c is not None else None, d_out.data_ptr(),
                                                      d_out.numel(), d_size.data_ptr(), words.data_ptr(), stream), "cl_shard_phase3")
        verdict = seam_verdict(gather_rows(words, group))
        mark(5)
        self.events = ev
        return verdict

    def encode_protected(self, d_in, d_out, d_size, group=None):
        """The copy-mode path (density_b200_cl_shard_prot_*): the arguments of encode, any input. The shard at the stream start runs the
        staged copy-map iteration in phase 1; then the round budget of the iteration runs on all ranks with torch.distributed exchanges
        (round words, P tables, C tables, transfers) and the device folds. Returns seam_verdict's (flags, total, offsets) over all ranks;
        flags != 0 only when an iteration did not settle, the automaton left the candidate states, or on an error: the pieces are then
        void."""
        rank, world = _rank_world(group)
        stream = _stream()
        dev = d_in.device
        lib = self._lib

        def check(rc, what):
            _check(rc, f"cl_shard_prot_{what}")

        n = d_in.numel()
        offset = int(gather_rows(torch.tensor([n], dtype=torch.int64, device=dev), group)[:rank].sum())
        words = torch.zeros(CL_PROT_ROUND_WORDS, dtype=torch.int32, device=dev)
        tp = torch.zeros(self.words_p, dtype=torch.int32, device=dev)
        tc = torch.zeros(self.words_c, dtype=torch.int32, device=dev)
        transfer = torch.zeros(PROT_TRANSFER_WORDS, dtype=torch.int32, device=dev)
        check(lib.density_b200_cl_shard_prot_phase1(self._h, d_in.data_ptr(), n, offset, int(rank == world - 1), words.data_ptr(), stream),
              "phase1")
        all_words = gather_rows(words, group).contiguous()
        for _ in range(lib.density_b200_prot_round_budget()):
            check(lib.density_b200_cl_shard_prot_p(self._h, all_words.data_ptr(), world, rank, tp.data_ptr(), stream), "p")
            carry_p = fold_cl_tables(self.alg, CL_TABLE_P, gather_rows(tp, group), rank)
            check(lib.density_b200_cl_shard_prot_c(self._h, carry_p.data_ptr(), tc.data_ptr(), stream), "c")
            carry_c = fold_cl_tables(self.alg, CL_TABLE_C, gather_rows(tc, group), rank)
            check(lib.density_b200_cl_shard_prot_transfer(self._h, carry_c.data_ptr(), transfer.data_ptr(), stream), "transfer")
            all_transfers = gather_rows(transfer, group).contiguous()
            check(lib.density_b200_cl_shard_prot_settle(self._h, all_transfers.data_ptr(), world, rank, words.data_ptr(), stream), "settle")
            all_words = gather_rows(words, group).contiguous()
            check(lib.density_b200_cl_shard_prot_next(self._h, all_words.data_ptr(), world, stream), "next")
        seam = torch.empty(SEAM_WORDS, dtype=torch.int32, device=dev)
        check(lib.density_b200_cl_shard_prot_finish(self._h, d_out.data_ptr(), d_out.numel(), d_size.data_ptr(), seam.data_ptr(), stream),
              "finish")
        return seam_verdict(gather_rows(seam, group))

    def prot_status(self):
        """density_b200_cl_shard_prot_status after encode_protected (waits for the device): dict with stage_settled (the staged
        iteration of the shard at the stream start settled; True elsewhere), rounds (until the map settled, 0: not settled), in_state
        ((penalty, start, previous_incompressible) entering the shard, None: left the candidates), esc and changed (this shard's blocks
        whose copy status changed, per round, 16 values)."""
        out = (ctypes.c_uint32 * PROT_STATUS_WORDS)()
        _check(self._lib.density_b200_cl_shard_prot_status(self._h, out), "cl_shard_prot_status")
        v = list(out)
        ins = None if v[2] == 0xFFFFFFFF else (v[2] & 0xFF, (v[2] >> 8) & 0xFF, v[2] >> 16)
        return {"stage_settled": bool(v[0]), "rounds": v[1], "in_state": ins, "esc": v[3], "changed": v[4:20]}

    def phase_ms(self):
        """[phase 1, P exchange + fold, phase 2, C exchange + fold, phase 3 + seams] in ms, of the last encode(timing=True)"""
        torch.cuda.synchronize()
        return [self.events[k].elapsed_time(self.events[k + 1]) for k in range(5)]


class ShardedChameleonDecoder(_Handle):
    """Decode of this rank's piece through the shard phases, with torch.distributed for the exchanges (the mirror of
    ShardedChameleonEncoder)."""

    def __init__(self):
        self._open("density_b200_decode_shard_create", "density_b200_decode_shard_destroy")

    def decode(self, d_in, d_out, d_size, group=None):
        """d_in: CUDA uint8 tensor, this rank's piece (2-byte aligned); d_out: uint8 tensor of capacity d_out.numel() (4-byte aligned);
        d_size: int64[1]. Returns seam_verdict's (flags, total, offsets) over all ranks; flags != 0: the pieces are void."""
        rank, world = _rank_world(group)
        return self._decode_piece(d_in, d_out, d_size, rank == world - 1, group)

    def decode_protected(self, d_in, d_out, d_size, group=None):
        """Decode of a piece of any stream, copy-mode blocks included (density_b200_decode_shard_prot_*): the arguments of decode. The
        pieces' protection transfers are exchanged first, then the tables as in decode. Returns seam_verdict's (flags, total, offsets);
        flags != 0: the pieces are void (a transfer path that does not end on a cut, a malformed piece, output beyond capacity)."""
        rank, world = _rank_world(group)
        stream = _stream()
        dev = d_in.device
        lib = self._lib
        transfer = torch.empty(DECODE_PROT_TRANSFER_WORDS, dtype=torch.int32, device=dev)
        _check(lib.density_b200_decode_shard_prot_transfer(self._h, d_in.data_ptr(), d_in.numel(), d_out.numel(), int(rank == world - 1),
                                                           transfer.data_ptr(), stream), "decode_shard_prot_transfer")
        self._transfers = gather_rows(transfer, group).contiguous()
        table = torch.empty(TABLE_ENTRIES, dtype=torch.int32, device=dev)
        _check(lib.density_b200_decode_shard_prot_phase1(self._h, self._transfers.data_ptr(), world, rank, table.data_ptr(), stream),
               "decode_shard_prot_phase1")
        gathered = gather_rows(table, group)
        carry_ptr = None
        if rank > 0:
            self._carry = fold_tables(gathered, rank)
            carry_ptr = self._carry.data_ptr()
        words = torch.empty(SEAM_WORDS, dtype=torch.int32, device=dev)
        _check(lib.density_b200_decode_shard_prot_phase2(self._h, carry_ptr, d_out.data_ptr(), d_size.data_ptr(), words.data_ptr(), stream),
               "decode_shard_prot_phase2")
        return seam_verdict(gather_rows(words, group))

    def decode_stream(self, d_in, n_range, d_out, d_size, group=None):
        """Decode of a stream without known cuts. d_in: CUDA uint8 tensor (2-byte aligned), this rank's range (its first n_range bytes)
        followed by its halo (stream_ranges gives the layout); d_out, d_size as in decode. Locates the piece (one host synchronisation
        for the maps) and decodes it. Returns (flags, total, offsets, my_offset): seam_verdict's result and where this rank's output
        starts in the original bytes; flags != 0: the pieces are void and the caller decodes the whole stream on one device."""
        rank = _rank_world(group)[0]
        n_halo = d_in.numel() - n_range
        if n_halo < 0:
            raise ValueError("d_in is shorter than its range")
        m = torch.empty(LOCATE_MAP_WORDS, dtype=torch.int64, device=d_in.device)
        _check(self._lib.density_b200_decode_locate(self._h, d_in.data_ptr(), n_range, n_halo, m.data_ptr(), _stream()), "decode_locate")
        maps = gather_rows(m, group)
        start, end, _, is_final = locate_piece(maps.cpu().numpy().view(np.uint64), rank)
        flags, total, offsets = self._decode_piece(d_in[start:end], d_out, d_size, bool(is_final), group)
        return flags, total, offsets, int(offsets[rank])

    def decode_stream_protected(self, d_in, n_range, d_out, d_size, group=None):
        """decode_stream for any stream, copy-mode blocks included: the protected range map (density_b200_decode_prot_locate), an
        all_gather of the maps (1.6 MiB per rank), prot_locate_piece on the host, then the located piece from its entry candidate
        (density_b200_decode_shard_prot_enter, prot_phase2). Returns (flags, total, offsets, my_offset) as decode_stream; a refused
        composition gives flags 1 on every rank without decoding."""
        rank, world = _rank_world(group)
        n_halo = d_in.numel() - n_range
        if n_halo < 0:
            raise ValueError("d_in is shorter than its range")
        m = torch.empty(PROT_LOCATE_MAP_WORDS, dtype=torch.int32, device=d_in.device)
        _check(self._lib.density_b200_decode_prot_locate(self._h, d_in.data_ptr(), n_range, n_halo, m.data_ptr(), _stream()),
               "decode_prot_locate")
        maps = gather_rows(m, group)
        start, end, is_final, _, cand, refused = prot_locate_piece(maps.cpu().numpy().view(np.uint32), rank)
        if refused:
            d_size.zero_()
            return 1, 0, torch.zeros(world + 1, dtype=torch.int64), 0
        flags, total, offsets = self._decode_piece(d_in[start:end], d_out, d_size, bool(is_final), group, cand)
        return flags, total, offsets, int(offsets[rank])

    def _decode_piece(self, d_in, d_out, d_size, is_last, group, cand=None):
        """cand: a located piece's entry candidate (the protected phases), None: the quiet phases"""
        rank = _rank_world(group)[0]
        stream = _stream()
        table = torch.empty(TABLE_ENTRIES, dtype=torch.int32, device=d_in.device)
        if cand is None:
            _check(self._lib.density_b200_decode_shard_phase1(self._h, d_in.data_ptr(), d_in.numel(), d_out.numel(), int(is_last),
                                                              table.data_ptr(), stream), "decode_shard_phase1")
        else:
            _check(self._lib.density_b200_decode_shard_prot_enter(self._h, d_in.data_ptr(), d_in.numel(), d_out.numel(), int(is_last), cand,
                                                                  table.data_ptr(), stream), "decode_shard_prot_enter")
        gathered = gather_rows(table, group)
        carry_ptr = None
        if rank > 0:
            self._carry = fold_tables(gathered, rank)
            carry_ptr = self._carry.data_ptr()
        words = torch.empty(SEAM_WORDS, dtype=torch.int32, device=d_in.device)
        phase2 = self._lib.density_b200_decode_shard_phase2 if cand is None else self._lib.density_b200_decode_shard_prot_phase2
        _check(phase2(self._h, carry_ptr, d_out.data_ptr(), d_size.data_ptr(), words.data_ptr(), stream),
               "decode_shard_phase2" if cand is None else "decode_shard_prot_phase2")
        return seam_verdict(gather_rows(words, group))


class _ShardedHandle(_Handle):
    """A `density_b200_sharded` handle: one process per GPU; the library owns its NCCL communicator (the 128-byte id travels once
    through torch.distributed). torch.distributed is only used to hand out the id."""

    def __init__(self, device, group=None):
        self.rank, self.world = _rank_world(group)
        ident = torch.zeros(128, dtype=torch.uint8)
        if self.world > 1:
            if self.rank == 0:
                buf = (ctypes.c_uint8 * 128)()
                _check(_lib.load().density_b200_sharded_unique_id(buf), "sharded_unique_id")
                ident = torch.tensor(list(buf), dtype=torch.uint8)
            t = ident.to(device) if dist.get_backend(group) == "nccl" else ident
            dist.broadcast(t, src=0, group=group)
            ident = t.cpu()
        self._id = ident.contiguous()
        self._open("density_b200_sharded_create", "density_b200_sharded_destroy", self._id.data_ptr() if self.world > 1 else None,
                   self.rank, self.world)
        self.d_total = torch.zeros(1, dtype=torch.int64, device=device)
        self.d_offset = torch.zeros(1, dtype=torch.int64, device=device)


class ShardedEncoder(_ShardedHandle):
    """The C++ multi-GPU path (`density_b200_encode_sharded`, include/density_b200.h): the table all-gather, the single fold kernel,
    the exact seam verdict and the optional variable-length gather of the pieces to one rank, over the library's NCCL communicator.
    """

    def encode(self, d_in, d_out, d_size, d_flags, gather_root=-1, d_gather=None, alg="chameleon"):
        """Enqueue on torch's current stream. d_size int64[1]: this rank's piece; d_flags int32[1]: != 0 -> the stream is not quiet and
        the pieces are void; self.d_total int64[1]: stream length. gather_root >= 0: pieces gathered into d_gather on that rank (blocks).
        alg "cheetah" / "lion" (or their ids): density_b200_encode_sharded_cl, the same contract for those algorithms."""
        args = (d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), d_out.numel(), d_size.data_ptr(), d_flags.data_ptr(), self.d_total.data_ptr(),
                int(gather_root), d_gather.data_ptr() if d_gather is not None else None, d_gather.numel() if d_gather is not None else 0, _stream())
        alg = _alg_id(alg)
        if alg == 0:
            rc = self._lib.density_b200_encode_sharded(self._h, *args)
        else:
            rc = self._lib.density_b200_encode_sharded_cl(self._h, alg, *args)
        _check(rc, f"encode_sharded{'' if alg == 0 else '_cl'}")

    def encode_protected(self, d_in, d_out, d_size, d_flags, gather_root=-1, d_gather=None, alg="chameleon"):
        """density_b200_encode_sharded_protected: Chameleon with copy mode, the arguments of encode. d_flags != 0 only when the copy map
        did not settle within the round budget, the automaton left the candidate states, or on an error: the pieces are then void.
        alg "cheetah" / "lion" (or their ids): density_b200_encode_sharded_cl_protected, the same contract for those algorithms (the call
        waits once for the gathered shard lengths)."""
        args = (d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), d_out.numel(), d_size.data_ptr(), d_flags.data_ptr(), self.d_total.data_ptr(),
                int(gather_root), d_gather.data_ptr() if d_gather is not None else None, d_gather.numel() if d_gather is not None else 0, _stream())
        alg = _alg_id(alg)
        if alg == 0:
            rc = self._lib.density_b200_encode_sharded_protected(self._h, *args)
        else:
            rc = self._lib.density_b200_encode_sharded_cl_protected(self._h, alg, *args)
        _check(rc, f"encode_sharded{'' if alg == 0 else '_cl'}_protected")

    def profile(self):
        """stage times (ms) of the last encode: Chameleon flag pass, table exchange + fold, carry / resolve / sizes / scan, emit, seams +
        gather; Cheetah / Lion phase 1, P exchange + fold, phase 2 + C exchange + fold, phase 3, seams + gather"""
        out = (ctypes.c_float * 5)()
        _check(self._lib.density_b200_sharded_profile(self._h, out), "sharded_profile")
        return [float(x) for x in out]


class ShardedDecoder(_ShardedHandle):
    """The C++ multi-GPU decode (`density_b200_decode_sharded`): the inverse of ShardedEncoder.encode without a gather. Each rank
    decodes its piece back into the shard it was encoded from; the exchanges run over the library's NCCL communicator."""

    def decode(self, d_in, d_out, d_size, d_flags, alg="chameleon"):
        """Enqueue on torch's current stream; nothing blocks. d_in: this rank's piece (2-byte aligned); d_out: capacity d_out.numel()
        (4-byte aligned); d_size int64[1]: the decoded size; d_flags int32[1]: != 0 -> the pieces are void and the caller decodes the
        gathered stream on one device; self.d_total int64[1]: the original length. alg "cheetah" (or its id): the pieces of a sharded
        Cheetah stream (density_b200_decode_sharded_cheetah). Lion pieces decode through ShardedLionDecoder."""
        alg = _alg_id(alg)
        if alg not in (0, 1):
            raise ValueError("sharded decode: alg must be 'chameleon' or 'cheetah' (Lion pieces decode through ShardedLionDecoder)")
        fn = self._lib.density_b200_decode_sharded if alg == 0 else self._lib.density_b200_decode_sharded_cheetah
        _check(fn(self._h, d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), d_out.numel(), d_size.data_ptr(), d_flags.data_ptr(),
                  self.d_total.data_ptr(), _stream()), f"decode_sharded{'' if alg == 0 else '_cheetah'}")

    def decode_protected(self, d_in, d_out, d_size, d_flags, alg="chameleon"):
        """density_b200_decode_sharded_protected: the Chameleon pieces of any stream, copy-mode blocks included (the inverse of
        ShardedEncoder.encode_protected), with the arguments of decode. Enqueued on torch's current stream; nothing blocks. alg
        "cheetah" (or its id): the Cheetah pieces of any stream (density_b200_decode_sharded_cheetah_protected, the inverse of
        ShardedEncoder.encode_protected(..., alg="cheetah"))."""
        alg = _alg_id(alg)
        if alg not in (0, 1):
            raise ValueError("sharded decode: alg must be 'chameleon' or 'cheetah' (Lion pieces decode through ShardedLionDecoder)")
        fn = self._lib.density_b200_decode_sharded_protected if alg == 0 else self._lib.density_b200_decode_sharded_cheetah_protected
        _check(fn(self._h, d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), d_out.numel(), d_size.data_ptr(), d_flags.data_ptr(),
                  self.d_total.data_ptr(), _stream()), f"decode_sharded{'' if alg == 0 else '_cheetah'}_protected")

    def decode_stream(self, d_in, n_range, d_out, d_size, d_flags, alg="chameleon", range_offset=None):
        """Decode of a stream without known cuts (`density_b200_decode_sharded_stream`). d_in: this rank's range (its first n_range
        bytes) followed by its halo (stream_ranges gives the layout); the rest as in decode. Blocks once, on the range maps.
        self.d_offset int64[1]: where this rank's output starts in the original bytes. alg "cheetah" (or its id): a Cheetah stream
        (density_b200_decode_sharded_cheetah_stream); range_offset, where this rank's range starts in the stream, is then required."""
        alg = _alg_id(alg)
        if alg not in (0, 1):
            raise ValueError("sharded stream decode: alg must be 'chameleon' or 'cheetah' (Lion streams without known cuts are decoded on one device)")
        if alg == 1 and range_offset is None:
            raise ValueError("sharded Cheetah stream decode: range_offset is required")
        n_halo = d_in.numel() - n_range
        tail = (d_out.data_ptr(), d_out.numel(), d_size.data_ptr(), self.d_offset.data_ptr(), d_flags.data_ptr(), self.d_total.data_ptr(), _stream())
        if alg == 0:
            rc = self._lib.density_b200_decode_sharded_stream(self._h, d_in.data_ptr(), n_range, n_halo, *tail)
        else:
            rc = self._lib.density_b200_decode_sharded_cheetah_stream(self._h, d_in.data_ptr(), n_range, n_halo, int(range_offset), *tail)
        _check(rc, f"decode_sharded{'' if alg == 0 else '_cheetah'}_stream")

    def decode_stream_protected(self, d_in, n_range, d_out, d_size, d_flags, alg="chameleon"):
        """decode_stream for any stream, copy-mode blocks included (density_b200_decode_sharded_stream_protected, or with alg "cheetah"
        density_b200_decode_sharded_cheetah_stream_protected, which needs no range offset). The arguments and outputs of decode_stream;
        blocks once, on the composition of the range maps. A refused composition sets d_flags to 1 on every rank."""
        alg = _alg_id(alg)
        if alg not in (0, 1):
            raise ValueError("sharded stream decode: alg must be 'chameleon' or 'cheetah' (Lion streams without known cuts are decoded on one device)")
        n_halo = d_in.numel() - n_range
        if n_range < 0 or n_halo < 0:
            raise ValueError("d_in is shorter than its range")
        fn = self._lib.density_b200_decode_sharded_stream_protected if alg == 0 else self._lib.density_b200_decode_sharded_cheetah_stream_protected
        _check(fn(self._h, d_in.data_ptr(), n_range, n_halo, d_out.data_ptr(), d_out.numel(), d_size.data_ptr(), self.d_offset.data_ptr(),
                  d_flags.data_ptr(), self.d_total.data_ptr(), _stream()), f"decode_sharded{'' if alg == 0 else '_cheetah'}_stream_protected")


class ShardedLionDecoder(_ShardedHandle):
    """The C++ multi-GPU Lion decode (`density_b200_decode_sharded_lion`): the inverse of ShardedEncoder.encode(..., alg="lion") without
    a gather. Boundaries, unpack and the chunk map run on every rank at once; the prediction walk is relayed from rank to rank, so the
    pieces walk one after the other and the whole decode takes about as long as decoding the stream on one device."""

    def decode(self, d_in, d_out, d_size, d_flags):
        """Enqueue on torch's current stream; nothing blocks. d_in: this rank's piece (2-byte aligned); d_out: capacity d_out.numel()
        (4-byte aligned); d_size int64[1]: the decoded size; d_flags int32[1]: != 0 -> the pieces are void and the caller decodes the
        gathered stream on one device; self.d_total int64[1]: the original length."""
        _check(self._lib.density_b200_decode_sharded_lion(self._h, d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), d_out.numel(),
                                                          d_size.data_ptr(), d_flags.data_ptr(), self.d_total.data_ptr(), _stream()),
               "decode_sharded_lion")

    def decode_protected(self, d_in, d_out, d_size, d_flags):
        """density_b200_decode_sharded_lion_protected: the Lion pieces of any stream, copy-mode blocks included (the inverse of
        ShardedEncoder.encode_protected(..., alg="lion")), with the arguments of decode."""
        _check(self._lib.density_b200_decode_sharded_lion_protected(self._h, d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), d_out.numel(),
                                                                    d_size.data_ptr(), d_flags.data_ptr(), self.d_total.data_ptr(), _stream()),
               "decode_sharded_lion_protected")
