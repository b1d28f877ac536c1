// encode_internal.cuh — host-side interfaces between api.cu and the kernel translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

namespace dns {

// chameleon_encode.cu
// byte offsets of the Chameleon encode scratch arrays inside one workspace allocation
struct ChamLayout {
    size_t status, sigw, copymap, copymap2, seg_state, incb, tile_bytes, tile_local, group_total, group_off, unres, unres_count, final_tab, carry, total;
};

size_t cham_workspace_bytes(size_t nbytes, int nruns_max, ChamLayout* L);
uint32_t cham_pick_runs(size_t nbytes, int num_sms);
cudaError_t cham_encode_phase1(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns,
                               uint32_t* d_table_out, cudaStream_t stream, uint64_t* launches, cudaEvent_t* ev = nullptr);
cudaError_t cham_encode_phase2(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns,
                               const uint32_t* d_carry_in, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                               bool allow_protected_fallback, bool assume_prev_inc, int num_sms, cudaStream_t stream, uint64_t* launches,
                               cudaEvent_t* ev = nullptr);
cudaError_t cham_encode_phase2_blocking(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns, uint8_t* d_out,
                                        size_t cap, uint64_t* d_out_size, int max_batches, int num_sms, cudaStream_t stream, uint64_t* launches);
cudaError_t cham_encode_protected_only(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint8_t* d_out,
                                       size_t cap, uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches);

// streaming continuation (a reused Codec instance, codec.rs:16,72): the dictionary as the reference keeps it (65536 quads) <-> the
// touched | fingerprint form of the run-parallel encoder; and phase 2 with a carried-in dictionary that gives up (no emit, *ok = false)
// instead of walking in order when the copy map does not settle
cudaError_t cham_quads_to_table(const uint32_t* d_quads, uint32_t* d_table, cudaStream_t stream, uint64_t* launches);
cudaError_t cham_table_into_quads(const uint32_t* d_table, uint32_t* d_quads, cudaStream_t stream, uint64_t* launches);
cudaError_t cham_encode_phase2_stream(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns, const uint32_t* d_carry_in,
                                      uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_table_out, int max_batches, int num_sms,
                                      cudaStream_t stream, uint64_t* launches, bool* ok);

// table helpers (sharded API, pipelined host path)
cudaError_t cham_status_accumulate(const uint8_t* ws, const ChamLayout& L, uint32_t* d_flag, cudaStream_t stream, uint64_t* launches);
cudaError_t cham_table_init(uint32_t* d_table, cudaStream_t stream, uint64_t* launches);
cudaError_t cham_rank_fold(const uint32_t* d_tables, uint32_t rank, uint32_t* d_carry, cudaStream_t stream, uint64_t* launches);
cudaError_t cham_seam_words(const uint8_t* ws, const ChamLayout& L, size_t nbytes, const uint64_t* d_out_size, uint32_t* d_words, cudaStream_t stream, uint64_t* launches);
cudaError_t cham_seam_verdict(const uint32_t* d_all_words, uint32_t world, uint32_t rank, uint32_t* d_flags, uint64_t* d_total, uint64_t* d_offsets,
                              cudaStream_t stream, uint64_t* launches);
cudaError_t cham_table_fold(uint32_t* d_acc, const uint32_t* d_next, cudaStream_t stream, uint64_t* launches);

// shared pieces of the encoders (chameleon_encode.cu)
struct Status;
size_t prot_state_bytes(uint64_t nseg_max);   // segment states + candidate tables of prot_iterate for up to nseg_max segments of 256 blocks
cudaError_t prot_debug_read(unsigned long long* out32);   // diagnostics: per fixed-point round {first changed block, changed blocks}
cudaError_t prot_iterate_launch(const uint32_t* sigw_or_null, uint64_t nbytes, uint64_t nblocks, uint32_t nseg, Status* st, int it, uint8_t* inc,
                                uint8_t* cm_old, uint8_t* cm_new, uint32_t* in_state, uint32_t* out_state, int num_sms, cudaStream_t stream);
cudaError_t scan_tiles_launch(const uint32_t* tile_bytes, uint32_t ntiles, uint32_t* tile_local, uint64_t* group_total, uint64_t* group_off,
                              uint32_t ngroups, Status* st, uint64_t cap, uint64_t* d_out_size, cudaStream_t stream);

// sharded copy-map iteration (density_b200_shard_prot_*): one shard of a longer stream. The shard's record lives in device memory.
struct ProtShard {
    unsigned long long first_block;   // global index of the shard's first block
    uint32_t rounds;                  // rounds run until the map settled (0: not settled)
    uint32_t settled, in_state, esc;  // in_state: pc_encode candidate of the true incoming state of the last round (0xFFFF: PC_ESC)
    uint32_t changed[16];             // blocks of this shard whose copy status changed, per round
    uint32_t stage_ok;                // 0: the shard's own staged iteration did not settle (Cheetah / Lion, the shard at the stream start)
    uint32_t has_quad, last_quad;     // Cheetah / Lion: the shard's last encoded quad under the map of the next round, if it has one
};
constexpr uint32_t PROT_TRANSFER_WORDS = 200, PROT_ROUND_WORDS = 4, PROT_MAX_ROUNDS = 16;
// The launches of the sharded copy-map iteration that every codec shares, on one shard's blocks (nblocks of the codec's size): the
// incompressible bits `inc`, the committed map `cm`, the next map `cm2`, and the segment states and candidate tables in a region of
// prot_state_bytes(). Round words are rows of `stride` u32 that start {changed, met PC_ESC, settled before this round, 0}.
struct ProtSegs {
    Status* st; uint64_t nbytes, nblocks; uint32_t nseg, ngrp;
    uint8_t *inc, *cm, *cm2; uint32_t *in_state, *gin; uint16_t *T, *GT;
};
ProtSegs prot_segs(Status* st, uint64_t nbytes, uint64_t nblocks, uint8_t* inc, uint8_t* cm, uint8_t* cm2, uint32_t* seg_state);
// the record of a shard that starts at first_block (or at the sum of d_lengths[0 .. rank) / block_bytes); opens the gate of the rounds
cudaError_t prot_start(const ProtSegs& P, ProtShard* ps, uint64_t first_block, const uint64_t* d_lengths, uint32_t rank, uint32_t block_bytes,
                       cudaStream_t stream, uint64_t* launches);
// the shard's transfer (PROT_TRANSFER_WORDS u32); sigw: Chameleon's signatures, from which the bits are refreshed first (nullptr: as they are)
cudaError_t prot_transfer(const ProtSegs& P, const uint32_t* sigw, const ProtShard* ps, int it, uint32_t* d_transfer_out, cudaStream_t stream,
                          uint64_t* launches);
// the true incoming state from the transfers of the shards before `rank`, the walk into cm2, words 0-3 of d_words. warm: round 0's flags
// were computed under cm (else under the empty map)
cudaError_t prot_settle(const ProtSegs& P, ProtShard* ps, int it, int warm, const uint32_t* d_all_transfers, uint32_t rank, uint32_t* d_words,
                        cudaStream_t stream, uint64_t* launches);
// the global commit and verdict of round `it` from the gathered round words
cudaError_t prot_commit(const ProtSegs& P, ProtShard* ps, int it, const uint32_t* d_all_words, uint32_t world, uint32_t stride, cudaStream_t stream,
                        uint64_t* launches);
// before the emit: the error of a shard that did not settle; after it: the 8 seam words (word 2: refused or error; the size is then 0)
cudaError_t prot_refuse_unsettled(Status* st, const ProtShard* ps, cudaStream_t stream, uint64_t* launches);
cudaError_t prot_seam_words(uint64_t nblocks, Status* st, uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t stream, uint64_t* launches);
// start: after cham_encode_phase1 (round 0's flags); first_block, or the sum of lengths[0 .. rank) / 256 when d_lengths is set
cudaError_t cham_prot_start(uint8_t* ws, const ChamLayout& L, ProtShard* ps, uint64_t first_block, const uint64_t* d_lengths, uint32_t rank,
                            cudaStream_t stream, uint64_t* launches);
cudaError_t cham_put_u64(uint64_t* d, uint64_t v, cudaStream_t stream, uint64_t* launches);   // *d = v in stream order
// round `it`: resolve the flags against the carry-in (NULL = stream start), export the transfer (PROT_TRANSFER_WORDS u32)
cudaError_t cham_prot_transfer(size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns, const uint32_t* d_carry_in, const ProtShard* ps,
                               int it, uint32_t* d_transfer_out, cudaStream_t stream, uint64_t* launches);
// compose the gathered transfers of the shards before `rank`, walk, compare: PROT_ROUND_WORDS u32 to d_words
cudaError_t cham_prot_settle(size_t nbytes, uint8_t* ws, const ChamLayout& L, ProtShard* ps, int it, const uint32_t* d_all_transfers, uint32_t rank,
                             uint32_t* d_words, cudaStream_t stream, uint64_t* launches);
// the global commit of round `it` from the gathered round words; with d_table_out, round it + 1's flags under the new map and its table
cudaError_t cham_prot_next(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns, ProtShard* ps, int it,
                           const uint32_t* d_all_words, uint32_t world, uint32_t* d_table_out, cudaStream_t stream, uint64_t* launches);
// sizes under the copy map, scan, emit, 8 seam words (word 2: refused or error); ev as cham_encode_phase2
cudaError_t cham_prot_finish(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, const ProtShard* ps, uint8_t* d_out, size_t cap,
                             uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t stream, uint64_t* launches, cudaEvent_t* ev = nullptr);

// cheetah_encode.cu
extern int g_chee_stage_rounds;
size_t chee_workspace_bytes(size_t nbytes, int num_sms);
size_t chee_tables_bytes(int alg, int region, size_t nbytes, int num_sms);
cudaError_t chee_encode_parallel(int alg, const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, uint8_t* const tables[3],
                                 uint32_t epoch_base, int num_sms, uint64_t* d_out_size, uint32_t* d_converged, bool resume,
                                 cudaStream_t stream, uint64_t* launches);
// sharded Cheetah / Lion encode: one shard of a longer stream (non-final shards whole 256-byte multiples). Tables are stacks of
// cl_table_planes(alg, kind) planes of 65536 u32 (kind 0 = predictions, 1 = chunk map). Every phase of one shard gets the same record:
// the shard d_in[0 .. n) at byte `offset` of the stream; first: the shard at the stream start, which alone may use copy mode (quiet
// phases: the shard without a d_prev_quad; prot phases: offset 0 and n > 0); last: no stream byte follows it; ws and the three tables
// (chee_tables_bytes regions); the epochs from epoch_base; ps: the record of the copy-map iteration (device, prot phases only).
struct ClShardArgs { int alg; const uint8_t* d_in; size_t n; uint64_t offset; bool first, last; uint8_t* ws; uint8_t* tables[3]; uint32_t epoch_base;
                     int num_sms; ProtShard* ps; };
// Each quiet phase 1 takes cl_shard_epochs() fresh epochs; phases 2 and 3 get the same epoch_base. d_prev_quad: the last quad of the
// stream before the shard (nullptr for the first shard); d_carry_*: the carried-in state (nullptr = stream start).
uint32_t cl_shard_epochs();
uint32_t cl_table_planes(int alg, int kind);
size_t cl_shard_workspace_bytes(size_t nbytes, int num_sms);
cudaError_t cl_shard_phase1(const ClShardArgs& a, const uint32_t* d_prev_quad, uint32_t* d_tab_p, cudaStream_t stream, uint64_t* launches);
cudaError_t cl_shard_phase2(const ClShardArgs& a, const uint32_t* d_carry_p, uint32_t* d_tab_c, cudaStream_t stream, uint64_t* launches);
cudaError_t cl_shard_phase3(const ClShardArgs& a, const uint32_t* d_carry_c, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8,
                            cudaStream_t stream, uint64_t* launches);
cudaError_t cl_table_init(int alg, int kind, uint32_t* d_table, cudaStream_t stream, uint64_t* launches);
cudaError_t cl_table_fold(int alg, int kind, uint32_t* d_acc, const uint32_t* d_next, cudaStream_t stream, uint64_t* launches);
cudaError_t cl_rank_fold(int alg, int kind, const uint32_t* d_tables, uint32_t rank, uint32_t* d_carry, cudaStream_t stream, uint64_t* launches);
cudaError_t cl_last_quad(const uint8_t* d_in, size_t n, uint32_t* d_out2, cudaStream_t stream, uint64_t* launches);   // {has a quad, last quad}
cudaError_t cl_prev_quad(const uint32_t* d_words, uint32_t rank, uint32_t* d_out, cudaStream_t stream, uint64_t* launches);
// the same with copy-mode blocks anywhere (density_b200_cl_shard_prot_*): the copy-map iteration carried over the cuts, round for round.
// The first shard runs the staged iteration in phase 1; each prot phase 1 takes cl_prot_epochs() fresh epochs from epoch_base. Round
// words: CL_PROT_ROUND_WORDS u32, {changed, met PC_ESC, settled before, 0, has an encoded quad, that quad, 0, 0}.
constexpr uint32_t CL_PROT_ROUND_WORDS = 8;
uint32_t cl_prot_epochs();
cudaError_t cl_prot_phase1(const ClShardArgs& a, uint32_t* d_words8, cudaStream_t stream, uint64_t* launches);
cudaError_t cl_prot_p(const ClShardArgs& a, int it, const uint32_t* d_all_words, uint32_t rank, uint32_t* d_tab_p, cudaStream_t stream,
                      uint64_t* launches);
cudaError_t cl_prot_c(const ClShardArgs& a, int it, const uint32_t* d_carry_p, uint32_t* d_tab_c, cudaStream_t stream, uint64_t* launches);
cudaError_t cl_prot_transfer(const ClShardArgs& a, int it, const uint32_t* d_carry_c, uint32_t* d_transfer, cudaStream_t stream, uint64_t* launches);
cudaError_t cl_prot_settle(const ClShardArgs& a, int it, const uint32_t* d_all_transfers, uint32_t rank, uint32_t* d_words8, cudaStream_t stream,
                           uint64_t* launches);
cudaError_t cl_prot_next(const ClShardArgs& a, int it, const uint32_t* d_all_words, uint32_t world, cudaStream_t stream, uint64_t* launches);
// ev_emit (may be nullptr): recorded between the scan and the emit
cudaError_t cl_prot_finish(const ClShardArgs& a, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t stream,
                           uint64_t* launches, cudaEvent_t ev_emit = nullptr);

// chameleon_decode.cu
size_t cham_decode_workspace_bytes(size_t nbytes, size_t cap, int nruns_max);
cudaError_t cham_decode_parallel(const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, int num_sms,
                                 uint64_t* d_out_size, uint32_t* d_nonquiet, cudaStream_t stream, uint64_t* launches);
// the same as two phases, for one piece of a sharded stream: phase 1 needs no carry-in and exports the piece's last-writer table
// (shard format) when d_table_out is set; phase 2 decodes from d_carry_in (NULL: stream start); then the piece's 8 seam words
// d_seed (may be NULL): the piece's incoming automaton state (cham_decode_prot_enter); rows_ready: cham_decode_prot_transfer on the same
// workspace filled the candidate rows
cudaError_t cham_decode_phase1(const uint8_t* d_in, size_t nbytes, size_t cap, uint8_t* ws, int num_sms, uint32_t* d_table_out,
                               cudaStream_t stream, uint64_t* launches, const uint32_t* d_seed = nullptr, bool rows_ready = false);
cudaError_t cham_decode_phase2(const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, int num_sms, const uint32_t* d_carry_in,
                               uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches);
cudaError_t cham_decode_seam_words(const uint8_t* d_in, size_t nbytes, size_t cap, uint8_t* ws, int num_sms, int is_last, const uint64_t* d_out_size,
                                   uint32_t* d_words, cudaStream_t stream, uint64_t* launches);
// a piece of a stream with copy-mode blocks: its protection transfer (DECODE_PROT_TRANSFER_WORDS, fills the candidate rows of the workspace
// first), its incoming state composed from candidate x0 and the transfers of the pieces before it (DECODE_PROT_SEED_WORDS), and its seam
// words after cham_decode_phase1 with that seed and cham_decode_phase2 (nbytes 0: an empty piece, the workspace is not read)
constexpr uint32_t DECODE_PROT_TRANSFER_WORDS = 3200, DECODE_PROT_SEED_WORDS = 5;
cudaError_t cham_decode_prot_transfer(const uint8_t* d_in, size_t nbytes, uint8_t* ws, int is_last, uint32_t* d_transfer, cudaStream_t stream,
                                      uint64_t* launches);
cudaError_t cham_decode_prot_enter(const uint32_t* d_all_transfers, uint32_t rank, uint32_t x0, uint32_t* d_seed, cudaStream_t stream,
                                   uint64_t* launches);
cudaError_t cham_decode_prot_seam_words(size_t nbytes, size_t cap, uint8_t* ws, int num_sms, int is_last, const uint32_t* d_seed, uint64_t* d_out_size,
                                        uint32_t* d_words, cudaStream_t stream, uint64_t* launches);
// the range map of a piece of a stream without known cuts (DENSITY_B200_LOCATE_MAP_WORDS u64 to d_map); scratch in `ws`, at least
// cham_locate_workspace_bytes(n_range + n_halo), which cham_decode_workspace_bytes of the same length covers
size_t cham_locate_workspace_bytes(size_t nbytes);
cudaError_t cham_decode_locate(const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* ws, uint64_t* d_map, cudaStream_t stream,
                               uint64_t* launches);
// the protected range map (DENSITY_B200_PROT_LOCATE_MAP_WORDS u32 to d_map), the same scratch
cudaError_t cham_decode_prot_locate(const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* ws, uint32_t* d_map, cudaStream_t stream,
                                    uint64_t* launches);

// cl_decode.cu (run-parallel Cheetah decode; parallel Lion decode with the prediction walk)
size_t chee_decode_workspace_bytes(size_t nbytes, size_t cap, int num_sms);
size_t chee_decode_tables_bytes(size_t nbytes, int num_sms, bool lion = false);
cudaError_t chee_decode_parallel(const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, uint8_t* tables, uint8_t* tail_ws,
                                 int num_sms, uint64_t* d_out_size, uint32_t* d_fallback, cudaStream_t stream, uint64_t* launches);
const void* chee_decode_status_ptr(uint8_t* ws, size_t nbytes, size_t cap, int num_sms, const void** cl_status);
// Lion: the same workspace contract (tables: chee_decode_tables_bytes(.., true)); the walk status behind *walk_status is a ClStatus prefix
// followed by 4 u64 counts {encoded quads, predicted quads, table reads that waited on a predicted quad, rows}
size_t lion_decode_workspace_bytes(size_t nbytes, size_t cap, int num_sms);
cudaError_t lion_decode_parallel(const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, uint8_t* tables, uint8_t* tail_ws,
                                 int num_sms, uint64_t* d_out_size, uint32_t* d_fallback, cudaStream_t stream, uint64_t* launches);
const void* lion_decode_status_ptr(uint8_t* ws, size_t nbytes, size_t cap, int num_sms, const void** walk_status);
// sharded Cheetah and Lion decode: one piece of a longer stream (first: it holds the stream start; last: no stream byte follows it; lion:
// the Lion geometry). ws holds chee_shard_workspace_bytes, tables chee_decode_tables_bytes of the piece. Phase 1 (or prot transfer, then
// phase 1 with the seed of chee_shard_prot_enter), phase 2, then Cheetah: any number of rounds (walk, exchange, fold); Lion: the walk; then
// phase 3. Every call of one piece gets the same arguments. Chunk-map tables: 3 planes {tags, a, b} of 65536 u32.
struct CheeShardArgs { const uint8_t* d_in; size_t n; uint8_t* d_out; size_t cap; bool first, last, lion; uint8_t* ws; uint8_t* tables; int num_sms; };
size_t chee_shard_workspace_bytes(size_t n, size_t cap, int num_sms, bool lion);
// d_seed (may be NULL): the piece's incoming automaton state (chee_shard_prot_enter); rows_ready: chee_shard_prot_transfer on the same
// workspace filled the candidate rows
cudaError_t chee_shard_phase1(const CheeShardArgs& a, uint32_t* d_cmap_out, cudaStream_t stream, uint64_t* launches, const uint32_t* d_seed = nullptr,
                              bool rows_ready = false);
cudaError_t chee_shard_phase2(const CheeShardArgs& a, const uint32_t* d_cmap_carry, cudaStream_t stream, uint64_t* launches);
// (d_seed: the same seed, whose seam words do not refuse incompressible blocks at the cuts; n == 0 is allowed there)
cudaError_t chee_shard_phase3(const CheeShardArgs& a, uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t stream, uint64_t* launches,
                              const uint32_t* d_seed = nullptr);
// a piece of a stream with copy-mode blocks: its protection transfer (DECODE_PROT_TRANSFER_WORDS; fills the candidate rows of the workspace
// first) and its incoming state composed from the transfers of the pieces before it (DECODE_PROT_SEED_WORDS), for chee_shard_phase1
cudaError_t chee_shard_prot_transfer(const CheeShardArgs& a, uint32_t* d_transfer, cudaStream_t stream, uint64_t* launches);
cudaError_t chee_shard_prot_enter(const uint32_t* d_all_transfers, uint32_t rank, uint32_t x0, uint32_t* d_seed, cudaStream_t stream,
                                  uint64_t* launches);
const void* chee_shard_status_ptr(const CheeShardArgs& a);
// Cheetah: the prediction rounds
uint32_t chee_shard_max_rounds();
cudaError_t chee_shard_round_walk(const CheeShardArgs& a, uint32_t round, uint32_t* d_pred_out, uint32_t* d_words, cudaStream_t stream, uint64_t* launches);
cudaError_t chee_shard_round_fold(const CheeShardArgs& a, uint32_t round, const uint32_t* d_pred_carry, const uint32_t* d_all_words, uint32_t world,
                                  uint32_t rank, cudaStream_t stream, uint64_t* launches);
cudaError_t chee_cmap_identity(uint32_t* d_table, cudaStream_t stream, uint64_t* launches);
cudaError_t chee_cmap_init(uint32_t* d_table, cudaStream_t stream, uint64_t* launches);
cudaError_t chee_cmap_fold(uint32_t* d_acc, const uint32_t* d_next, cudaStream_t stream, uint64_t* launches);
cudaError_t chee_cmap_rank_fold(const uint32_t* d_tables, uint32_t rank, uint32_t* d_carry, cudaStream_t stream, uint64_t* launches);
// Lion: the walk's state travels from piece to piece in LION_STATE_WORDS u32: the 65536 five-slot lists (the tail's layout), then
// last_hash, then padding.
constexpr uint32_t LION_STATE_WORDS = 5 * 65536 + 8;
cudaError_t lion_shard_walk(const CheeShardArgs& a, uint32_t* d_state, cudaStream_t stream, uint64_t* launches);
cudaError_t lion_state_init(uint32_t* d_state, cudaStream_t stream);
// the range map of a piece of a Cheetah stream without known cuts (DENSITY_B200_CHEETAH_LOCATE_MAP_WORDS u64 to d_map); scratch in `ws`,
// at least chee_locate_workspace_bytes of the same arguments
size_t chee_locate_workspace_bytes(size_t n_range, size_t n_halo, uint64_t range_offset);
cudaError_t chee_decode_locate(const uint8_t* d_in, size_t n_range, size_t n_halo, uint64_t range_offset, uint8_t* ws, uint64_t* d_map,
                               cudaStream_t stream, uint64_t* launches);
// the protected range map of any range (DENSITY_B200_CHEETAH_PROT_LOCATE_MAP_WORDS u32 to d_map); scratch chee_prot_locate_workspace_bytes(
// n_range + n_halo)
size_t chee_prot_locate_workspace_bytes(size_t nbytes);
cudaError_t chee_decode_prot_locate(const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* ws, uint32_t* d_map, cudaStream_t stream,
                                    uint64_t* launches);

// scalar_codec.cu (Cheetah / Lion, in-order)
size_t scalar_workspace_bytes(int alg);
cudaError_t scalar_encode(int alg, const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws,
                          uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches, const uint32_t* d_run_if_zero = nullptr, bool keep_state = false);
cudaError_t scalar_decode(int alg, const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws,
                          uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches, const uint32_t* d_run_if = nullptr, bool keep_state = false);
// tail loop only (codec.rs:102-123), Cheetah or Lion, continuing from the state the parallel decoder left: tables already in `ws`,
// boundary status (bounds::DecStatus: tail offset, block count, protection state) and the last hash (cheedec::ClStatus::final_ctx) on
// the device; runs only if *d_skip_if == 0
cudaError_t scalar_decode_tail(int alg, const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, const void* d_bounds_status,
                               const void* d_cl_status, uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches, const uint32_t* d_skip_if);

// decoded_size.cu: the length a stream decodes to, without decoding it; d_in 2-byte aligned, nbytes > 0. Writes {size, 0} or
// {0, DENSITY_B200_EMALFORMED} to d_result (2 x u64) in stream order; 4 kernels; scratch in `ws`, decoded_size_workspace_bytes(alg, nbytes)
size_t decoded_size_workspace_bytes(int alg, size_t nbytes);
cudaError_t decoded_size_launch(int alg, const uint8_t* d_in, size_t nbytes, uint8_t* ws, uint64_t* d_result, cudaStream_t stream,
                                uint64_t* launches);

// decode_range.cu: Chameleon range decode, d_in 2-byte aligned, nbytes > 0, len > 0. The locate step (4 kernels, scratch
// range_locate_workspace_bytes) writes {w, S, verdict} to d_result (3 x u64) and RANGE_REPORT_WORDS u64 to the workspace's start; the
// host reads them and range_plan turns them into the pieces (false: the report is inconsistent), whose decode range_decode_launch
// enqueues on a workspace of plan.ws_bytes (the report may be gone by then): 13 kernels for first < 256, else 26. *d_window: the w
// window bytes in that workspace, in stream order.
constexpr uint32_t RANGE_REPORT_WORDS = 8;
struct RangePlan {
    uint64_t w, k0, skip, off0, piece_n, stage_cap;    // skip: first - 256 k0, the window's offset in the staging
    uint32_t cand0;
    bool final_piece;
    size_t window_ws, ws_bytes;
    // an indexed piece (index_plan): the piece starts piece_off bytes into the stream and has its carry-in, carry_in (NULL: the stream
    // start); range_decode_launch then takes d_in at the piece and runs no prefix
    bool indexed;
    uint64_t piece_off;
    const uint32_t* carry_in;
};
size_t range_locate_workspace_bytes(size_t nbytes);
cudaError_t range_locate_launch(const uint8_t* d_in, size_t nbytes, uint64_t first, uint64_t len, uint8_t* ws, uint64_t* d_result,
                                cudaStream_t stream, uint64_t* launches);
bool range_plan(const uint64_t* report, size_t nbytes, uint64_t first, int num_sms, RangePlan* p);
cudaError_t range_decode_launch(const uint8_t* d_in, const RangePlan& p, uint8_t* ws, int num_sms, cudaStream_t stream, uint64_t* launches,
                                const uint8_t** d_window);

// The Chameleon seek index (DESIGN §4h, include/density_b200.h): a header of CIDX_HEADER_WORDS u64, a directory of C entries {u64 stream
// offset, u32 decode candidate, u32 0} padded to 256 bytes (with the header), then C snapshots of 65536 u32 in the shard table format.
constexpr uint64_t CIDX_MAGIC = 0x58444E494D414843ull;   // "CHAMINDX", little-endian
constexpr uint64_t CIDX_VERSION = 1, CIDX_HEADER_WORDS = 8, CIDX_SNAPSHOT_BYTES = 65536 * sizeof(uint32_t);
enum : uint32_t { CIDX_MAGIC_W, CIDX_VERSION_W, CIDX_N_W, CIDX_SIZE_W, CIDX_MAIN_BLOCKS_W, CIDX_INTERVAL_W, CIDX_COUNT_W, CIDX_BYTES_W };
__host__ __device__ inline uint64_t cidx_snapshots_at(uint64_t count) { return (CIDX_HEADER_WORDS * 8 + 16 * count + 255) & ~255ull; }
__host__ __device__ inline uint64_t cidx_bytes(uint64_t count) { return cidx_snapshots_at(count) + count * CIDX_SNAPSHOT_BYTES; }
// the most checkpoints an index of an n-byte stream can have at that interval (0 for an interval that is not a positive multiple of 256)
uint64_t index_max_count(size_t nbytes, uint64_t interval);
// Build, d_in 2-byte aligned, nbytes > 0: the locate step (4 kernels, scratch index_locate_workspace_bytes) writes {index bytes, S,
// verdict} to d_result and leaves index_report_bytes(index_max_count) bytes at the body of the workspace: the same three words, then the
// header and the directory, copied to h_report. The host waits for them; index_build_plan checks them (false: inconsistent) and sizes the
// workspace of index_build_launch, which writes the index to d_index (4-byte aligned): the header and the directory from h_report, then
// density_b200_table_init's state and per piece j = 0 .. C - 1 (j > 0: entered at checkpoint j's candidate) phase 1 with its table
// exported and a fold into snapshot j + 1: 14 C kernels (with the locate step, 4 + 14 C).
size_t index_report_bytes(uint64_t cmax);
size_t index_locate_workspace_bytes(size_t nbytes, uint64_t interval);
cudaError_t index_locate_launch(const uint8_t* d_in, size_t nbytes, uint64_t interval, uint8_t* ws, uint64_t* d_result, uint64_t* h_report,
                                cudaStream_t stream, uint64_t* launches);
bool index_build_plan(const uint64_t* report, size_t nbytes, int num_sms, size_t* ws_bytes);
cudaError_t index_build_launch(const uint8_t* d_in, const uint64_t* report, uint8_t* ws, uint8_t* d_index, int num_sms, cudaStream_t stream,
                               uint64_t* launches);
// Indexed range decode. index_count_for_bytes: the C whose layout is index_len bytes long (~0: none). index_check: NULL when the header
// and directory (host copy) are consistent with the stream length and index_len, else why not. index_plan: the piece of a window
// (false: first >= S, nothing to decode) and the checkpoint whose snapshot is its carry-in (0: none). range_table_slot: where a snapshot
// from host memory is staged. index_copy_out_launch: 1 kernel, the checked copy of the window to d_out (NULL: only the check) and the
// result words.
uint64_t index_count_for_bytes(uint64_t index_len);
const char* index_check(const uint64_t* hdr, size_t nbytes, uint64_t index_len, uint64_t count);
bool index_plan(const uint64_t* hdr, size_t nbytes, uint64_t first, uint64_t len, int num_sms, RangePlan* p, uint64_t* snapshot);
uint32_t* range_table_slot(uint8_t* ws);
cudaError_t index_copy_out_launch(const RangePlan& p, const uint8_t* d_window, uint64_t size, uint8_t* d_out, uint8_t* ws, uint64_t* d_result,
                                  int num_sms, cudaStream_t stream, uint64_t* launches);

}  // namespace dns
