/*
 * density_b200.h — C ABI of the H100-native (sm_90a) implementation of density's
 * Chameleon / Cheetah / Lion encode/decode hot path.
 *
 * Drop-in boundary. The first nine symbols have exactly the names, signatures and
 * semantics of the reference's own `extern "C"` exports, so a binary (or a Rust
 * `extern "C"` block, see INTEGRATION.md) that links against density-rs can link
 * against libdensity_b200.so instead:
 *
 *   chameleon_encode / chameleon_decode / chameleon_safe_encode_buffer_size
 *       replace /root/reference/src/algorithms/chameleon/chameleon.rs:70-83
 *   cheetah_encode / cheetah_decode / cheetah_safe_encode_buffer_size
 *       replace /root/reference/src/algorithms/cheetah/cheetah.rs:105-118
 *   lion_encode / lion_decode / lion_safe_encode_buffer_size
 *       replace /root/reference/src/algorithms/lion/lion.rs:193-206
 *
 * They take plain pointers and sizes. The pointers may be HOST pointers (pageable or
 * pinned; the library stages through device memory) or DEVICE pointers (detected with
 * cudaPointerGetAttributes; no staging). The call is synchronous and returns the number
 * of bytes written, or 0 on any error (the reference maps Err -> 0 the same way,
 * chameleon.rs:72 `unwrap_or(0)`; where the reference would panic on an undersized
 * buffer — io/write_buffer.rs:19 — this library returns 0 and never writes out of bounds).
 * Output is bit-identical to the reference's Codec::encode / Codec::decode
 * (codec/codec.rs:72-126) on the same input.
 *
 * There is no CPU fallback: every entry point fails (returns 0 / an error code) when no
 * CUDA device is usable.
 */
#ifndef DENSITY_B200_H
#define DENSITY_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define DENSITY_B200_API __attribute__((visibility("default")))
#else
#define DENSITY_B200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ---- the reference's FFI surface (host or device pointers, synchronous) ---------------- */
DENSITY_B200_API size_t chameleon_encode(const uint8_t* input, size_t input_size, uint8_t* output, size_t output_size);
DENSITY_B200_API size_t chameleon_decode(const uint8_t* input, size_t input_size, uint8_t* output, size_t output_size);
DENSITY_B200_API size_t chameleon_safe_encode_buffer_size(size_t size); /* codec/codec.rs:18-21 */

DENSITY_B200_API size_t cheetah_encode(const uint8_t* input, size_t input_size, uint8_t* output, size_t output_size);
DENSITY_B200_API size_t cheetah_decode(const uint8_t* input, size_t input_size, uint8_t* output, size_t output_size);
DENSITY_B200_API size_t cheetah_safe_encode_buffer_size(size_t size);

DENSITY_B200_API size_t lion_encode(const uint8_t* input, size_t input_size, uint8_t* output, size_t output_size);
/* PERFORMANCE LIMIT: lion_decode runs the parallel Lion decoder: boundaries, unpack and chunk-map values in parallel, then one warp
   walks the 5-deep prediction lists in stream order, 32 quads per step (DESIGN.md section 4c). That walk is serial over the whole
   stream: 0.05-0.22 GB/s measured on an H100 (README.md), 3.6-7x the in-order kernel but below the reference's CPU decoder, which
   stays the faster choice for large streams for this one symbol. Results are bit-exact. */
DENSITY_B200_API size_t lion_decode(const uint8_t* input, size_t input_size, uint8_t* output, size_t output_size);
DENSITY_B200_API size_t lion_safe_encode_buffer_size(size_t size);

/* ---- device-resident, stream-ordered variants (what bench.py times) --------------------- */
#define DENSITY_B200_CHAMELEON 0
#define DENSITY_B200_CHEETAH 1
#define DENSITY_B200_LION 2

#define DENSITY_B200_OK 0
#define DENSITY_B200_ECUDA 1      /* a CUDA runtime call failed (see density_b200_last_error) */
#define DENSITY_B200_ECAPACITY 2  /* output buffer too small */
#define DENSITY_B200_EMALFORMED 3 /* truncated / malformed stream on decode */
#define DENSITY_B200_EARG 4       /* bad argument (alignment, algorithm id, null pointer) */

/*
 * Encode `n` bytes at device pointer d_in (4-byte aligned) into d_out (2-byte aligned,
 * capacity `cap` >= *_safe_encode_buffer_size(n)). All work is enqueued on `stream`
 * (a cudaStream_t passed as void*; NULL = legacy default stream); nothing is synchronised.
 * The encoded size is written to *d_out_size (device memory, 8 bytes, 8-byte aligned) when the
 * stream reaches that point; it is 0 if the device-side capacity check failed. n == 0: no
 * kernel, 0 by a memset.
 * Returns DENSITY_B200_OK or an error code for failures detectable at enqueue time.
 * DENSITY_B200_EARG (a bad algorithm id, a NULL pointer, a misaligned d_out_size) enqueues nothing.
 */
DENSITY_B200_API int density_b200_encode_device(int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                               uint64_t* d_out_size, void* stream);
/*
 * Concurrent callers. The nine symbols above, the stream-ordered calls and the codec instances
 * on one device share one cached workspace (sharded handles have their own). Calls from
 * any host thread and on any stream are serialised on it in the order they are enqueued: a
 * call's device work starts when the previous call's work (on whatever stream) has finished
 * with the workspace. So a synchronous call (the nine symbols above, the codec instances)
 * waits for the stream-ordered calls enqueued before it, and returns only after they are done.
 * density_b200_shutdown must not overlap any other call.
 */
/* Test/diagnostic variant: choose the encode path explicitly.
   Chameleon: path 0 = auto (run-parallel fast path, exact protection-aware fallback when needed),
   1 = fast path only (no fallback; out size is only valid if the stream is "quiet"),
   2 = exact in-order protection-aware walk only, 3 = in-order single-thread kernel,
   4 = like 0, but the call may BLOCK on the stream: if the copy map has not settled after the 5 rounds that are always enqueued,
   the host keeps iterating (up to 96 more rounds) before the in-order walk takes over; this is what the nine reference
   symbols use (they are synchronous anyway).
   Cheetah / Lion: 0 = auto (run-parallel encoder; the in-order kernel, queued behind it, runs only if the copy map did
   not settle), 1 = run-parallel encoder only (*d_out_size == 0 if the copy map did not settle), 3 = in-order kernel,
   4 = like 0 but may BLOCK: the host reads the verdict and resumes the iteration (up to 12 times) before the in-order kernel. */
DENSITY_B200_API int density_b200_encode_device_path(int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                    uint64_t* d_out_size, void* stream, int path);
/* Decode counterpart: path 0 = auto (the parallel decoder of each algorithm, also for streams with copy-mode blocks; the exact
   in-order kernel is queued behind it as a safety net: it runs when the parallel decoder gives up — Cheetah: the context iteration
   did not settle; all: a malformed stream or a capacity error — and when d_in is not 2-byte or d_out not 4-byte aligned),
   1 = parallel decoder only (size 0 if it had to give up), 3 = in-order kernel only. */
DENSITY_B200_API int density_b200_decode_device_path(int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                    uint64_t* d_out_size, void* stream, int path);
/* Diagnostic: status of the last Chameleon encode on the current device (synchronises the device):
   out6 = {out_bytes, nonquiet (copy mode was needed), error, first_nonquiet_block, copy map converged, scratch}. */
DENSITY_B200_API int density_b200_encode_status(uint64_t* out6);
/* Diagnostic: status of the last parallel Chameleon decode on the current device (synchronises the device):
   out10 = {out_bytes, main_blocks, tail_off, nonquiet, error, last_main_inc, in_order_boundaries, penalty, penalty_start, prev_incompressible}.
   in_order_boundaries != 0: the stream had copy-mode blocks (codec.rs:89-92) and the boundaries came from the in-order walk. */
DENSITY_B200_API int density_b200_decode_status(uint64_t* out10);
/* Diagnostic: the context iteration of the last run-parallel Cheetah decode on the current device (synchronises the device):
   out4 = {rounds used, settled (0: the in-order kernel took over), run walks after round 0, round budget}. */
DENSITY_B200_API int density_b200_cheetah_decode_rounds(uint32_t* out4);
/* Diagnostic: the prediction walk of the last Lion decode on the current device (synchronises the device):
   out4 = {encoded quads walked, predicted quads, table reads that waited on a predicted quad, rows of 32 quads walked}.
   DENSITY_B200_EARG when that decode ran on the in-order kernel (path 3, misaligned buffers, codec instances) or there was none. */
DENSITY_B200_API int density_b200_lion_decode_stats(uint64_t* out4);
/* Same contract for decode; `cap` must be >= the original length. */
DENSITY_B200_API int density_b200_decode_device(int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                               uint64_t* d_out_size, void* stream);
/*
 * Decoded size: the number of bytes X::decode writes for a stream (the original length of an encoded input), found from the block
 * boundaries without decoding it. A stream does not record its length; this gives every decode entry point above the capacity it needs
 * for streams whose length the caller did not keep. Equivalent to decode for every byte string, whether or not an encoder wrote it:
 * a size s means decode with cap = s writes s bytes (and with cap = s - 1 writes 0); DENSITY_B200_EMALFORMED means decode writes 0 at
 * any capacity (the stream ends inside a block). A non-empty stream may decode to 0 bytes, hence the separate verdict.
 * Workspace: the boundary rows of the stream (3-7 % of n), independent of the decoded size; no output buffer.
 * Both calls use the device's shared workspace (see "Concurrent callers" above).
 *
 * Stream-ordered: d_in device, 2-byte aligned; d_result device, 8-byte aligned, receives two u64 {decoded size, verdict}, verdict 0 or
 * DENSITY_B200_EMALFORMED (then the size word is 0). n > 0: 4 kernels (the candidate rows, the in-order block walk, the tail); n == 0:
 * no kernel, {0, 0} by a memset. DENSITY_B200_EARG (a bad algorithm id, a NULL pointer, a misaligned d_in or d_result) enqueues nothing.
 */
DENSITY_B200_API int density_b200_decoded_size_device(int alg, const uint8_t* d_in, size_t n, uint64_t* d_result, void* stream);
/* Synchronous; host or device pointer of any alignment, like the nine reference symbols. DENSITY_B200_OK with *out_size set,
   DENSITY_B200_EMALFORMED, DENSITY_B200_EARG or DENSITY_B200_ECUDA. */
DENSITY_B200_API int density_b200_decoded_size(int alg, const uint8_t* input, size_t n, uint64_t* out_size);

/*
 * Chameleon range decode: bytes [first, first + len) of what a stream decodes to, without decoding the bytes in front of them and
 * without an output buffer of the decoded size. Let D = chameleon_decode(stream) with enough capacity and S = len(D). A range decode
 *   - writes w = min(first + len, S) - first bytes to d_out, or 0 bytes when first >= S, and those bytes are D[first : first + w];
 *   - writes nothing outside [d_out, d_out + w); d_out may have any alignment;
 *   - writes 0 bytes and reports DENSITY_B200_EMALFORMED when the stream is malformed, in the sense of density_b200_decoded_size (decode
 *     writes 0 at any capacity). The check covers the whole stream, not only the blocks in front of the window, so a window is always
 *     a slice of what decode returns.
 * Chameleon's state at a block boundary depends on no decoded value: the dictionary in front of block k holds the last PLAIN quad
 * before k of each bucket, and the protection automaton reads signatures only. So the call walks the block boundaries of the whole
 * stream (as density_b200_decoded_size does), rebuilds the dictionary in front of block k0 = first / 256 from the PLAIN quads of the
 * prefix (no decode pass, no output), and decodes blocks k0 .. k1 (k1: the block of the window's last byte) with the sharded decode's
 * piece machinery, entered in the located automaton state. Cost: about a boundary walk of the stream plus the prefix's writer pass plus
 * a decode of the window's blocks.
 * Scratch (the device's shared workspace): the boundary rows of the stream (3-7 % of n), the workspace of a decode of the blocks up to
 * k1 (block offsets, run tables) and staging for the window's decoded blocks, (k1 - k0 + 1) x 256 bytes, or S - 256 k0 when the window
 * ends in the tail loop's blocks (at most two blocks more). Nothing scales with S beyond block k1.
 * Cheetah and Lion have no range entry: their state at a block is the prediction map, keyed by the contexts of decoded quads, so the
 * state in front of a window costs a decode of the whole prefix, which would save neither time nor memory over decode itself.
 *
 * Stream-ordered: d_in device, 2-byte aligned; d_out device, any alignment; d_result device, 8-byte aligned, receives three u64 {bytes
 * written w, S, verdict}, verdict 0 or DENSITY_B200_EMALFORMED (then w and S are 0). The call enqueues the boundary walk (4 kernels),
 * then waits on `stream` for it, because the lengths of the pieces it decodes size their grids: it returns when the work enqueued on
 * `stream` before it and the walk are done, with the rest enqueued. Then, when w > 0: 13 kernels when first < 256, else 26, and one
 * copy. n == 0 or len == 0: no kernel, {0, 0, 0} by a memset (S is not computed). DENSITY_B200_EARG (a NULL pointer, a misaligned d_in
 * or d_result) enqueues nothing. The call uses the device's shared workspace (see "Concurrent callers" above).
 */
DENSITY_B200_API int density_b200_chameleon_decode_range_device(const uint8_t* d_in, size_t n, uint64_t first, uint64_t len, uint8_t* d_out,
                                                                uint64_t* d_result, void* stream);
/* Synchronous; host or device pointers of any alignment, like the nine reference symbols. DENSITY_B200_OK with *written = w,
   DENSITY_B200_EMALFORMED (*written = 0), DENSITY_B200_EARG or DENSITY_B200_ECUDA. */
DENSITY_B200_API int density_b200_chameleon_decode_range(const uint8_t* input, size_t n, uint64_t first, uint8_t* output, uint64_t len,
                                                         uint64_t* written);

/*
 * Chameleon seek index: the state a range decode needs in front of a window, recorded once per stream at fixed checkpoints, so that a
 * range decode reads and decodes only the stream between two checkpoints, at the same cost wherever the window is and however long the
 * stream is. A host-resident stream then sends only that piece over PCIe.
 *
 * Format (version 1). One contiguous, position-independent blob with no pointers in it, so it can be stored beside the stream and
 * loaded again; a pure function of (stream, interval). All fields little-endian.
 *   - header, 8 x u64: magic "CHAMINDX" (0x58444E494D414843), version 1, n (stream bytes), S (decoded size), main_blocks (the blocks of
 *     the decoder's main loop), interval (decoded bytes between checkpoints, a positive multiple of 256; I = interval / 256 blocks), C
 *     (the checkpoint count) and the index's length in bytes;
 *   - checkpoints at blocks j x I, j = 1 .. C, with C x I < main_blocks (every checkpoint is inside the main loop; the stream start is
 *     the implicit checkpoint 0);
 *   - directory, C entries of 16 bytes {u64 stream offset of block j x I, u32 decode candidate (the automaton state in front of it, < 3200,
 *     as the sharded decode numbers them), u32 0}; the header and the directory together are padded with zeros to a multiple of 256 bytes;
 *   - snapshots, C x 65536 u32 (256 KiB each) in the shard table format (bit 16 touched, bits 0-15 fingerprint): snapshot j is
 *     density_b200_table_init's state folded with the last-writer tables of the pieces in front of checkpoint j, the dictionary in front
 *     of block j x I.
 * Length: ceil256(64 + 16 C) + 262144 C bytes.
 */
/* An upper bound of the index's length for any stream of n bytes at that interval (from n alone: the largest block count n bytes can
   hold); 0 when the interval is not a positive multiple of 256. */
DENSITY_B200_API uint64_t density_b200_chameleon_index_bytes(size_t n, uint64_t interval);
/* Builds the index of d_in[0 .. n) (device, 2-byte aligned, n > 0) into d_index (device, 4-byte aligned, index_cap bytes). d_result
   (device, 8-byte aligned) receives three u64 {index bytes, S, verdict}. On a malformed stream (in the sense of density_b200_decoded_size)
   it returns DENSITY_B200_EMALFORMED with d_result = {0, 0, DENSITY_B200_EMALFORMED} and writes nothing to d_index. The call enqueues a
   boundary walk of the whole stream that stops at every checkpoint (4 kernels) and waits on `stream` for it; then 14 C kernels: per
   piece between checkpoints, its writer pass and a fold into the next snapshot. DENSITY_B200_EARG (index_cap <
   density_b200_chameleon_index_bytes(n, interval), n == 0, a bad interval, a NULL or misaligned pointer) enqueues nothing. The call uses
   the device's shared workspace (see "Concurrent callers" above): the boundary rows of the stream, then a decode workspace for one piece. */
DENSITY_B200_API int density_b200_chameleon_index_build_device(const uint8_t* d_in, size_t n, uint64_t interval, uint8_t* d_index, size_t index_cap,
                                                               uint64_t* d_result, void* stream);
/* Synchronous; host or device pointers of any alignment. DENSITY_B200_OK with *index_len set, DENSITY_B200_EMALFORMED, DENSITY_B200_EARG
   or DENSITY_B200_ECUDA. */
DENSITY_B200_API int density_b200_chameleon_index_build(const uint8_t* input, size_t n, uint64_t interval, uint8_t* index, size_t index_cap,
                                                        uint64_t* index_len);
/*
 * Indexed range decode: the contract of density_b200_chameleon_decode_range_device (d_out gets D[first : first + w] and nothing outside
 * [d_out, d_out + w), d_result = {w, S, verdict}), from the piece of the stream between the checkpoint at or in front of block first / 256
 * and the first checkpoint behind the window's last block (or the stream end when there is none, or the window reaches the main loop's
 * end or S). The piece is entered at its checkpoint's candidate with its snapshot as the carry-in, read in place from d_index.
 *   - The call first copies the header and the directory to the host (one copy, one wait on `stream`) and checks them: the magic, the
 *     version, n, index_len against the layout for C, the interval, offsets even, strictly increasing and < n, candidates < 3200,
 *     C x I < main_blocks and 256 main_blocks <= S <= 256 main_blocks + 528. A failure is DENSITY_B200_EARG: no kernel runs and nothing is
 *     written to d_out or d_result.
 *   - S and the verdict come from the index: a stream is not walked again. The decoded piece must have the size the index promises for
 *     it, (c_b - c_a) x interval, or S - 256 c_a I for the final piece; otherwise the call writes {0, S, DENSITY_B200_EMALFORMED} and
 *     leaves d_out untouched. That catches an index that does not match its stream. An index of another stream with the same structure
 *     (the same block boundaries and automaton states) is not caught: as with a wrong capacity, that is the caller's error. It never
 *     makes the call read or write outside the stream, the index, d_out or the workspace.
 *   - Kernels: 15 whenever w > 0 (the entry, the piece's phase 1 and phase 2, the checked copy), wherever the window is; 1 when first >= S
 *     (the result words). Workspace: the decode of the piece, at most the window plus 2 x interval of output; nothing grows with n.
 * Stream-ordered: d_in device, 2-byte aligned; d_index device, 4-byte aligned; d_out device, any alignment; d_result device, 8-byte
 * aligned. n == 0 or len == 0: no kernel, {0, 0, 0} by a memset (the index is not read).
 */
DENSITY_B200_API int density_b200_chameleon_decode_range_indexed_device(const uint8_t* d_in, size_t n, const uint8_t* d_index, size_t index_len,
                                                                        uint64_t first, uint64_t len, uint8_t* d_out, uint64_t* d_result,
                                                                        void* stream);
/* Synchronous; host or device pointers of any alignment for the stream, the index and the output. A host stream is staged only from
   the piece's first byte to its last; a host index only for its header, its directory and the one snapshot the piece starts from.
   DENSITY_B200_OK with *written = w, DENSITY_B200_EMALFORMED (*written = 0), DENSITY_B200_EARG or DENSITY_B200_ECUDA. */
DENSITY_B200_API int density_b200_chameleon_decode_range_indexed(const uint8_t* input, size_t n, const uint8_t* index, size_t index_len,
                                                                 uint64_t first, uint8_t* output, uint64_t len, uint64_t* written);

/*
 * Sharded encode. Every entry of the phase APIs of a Chameleon, Cheetah or Lion shard below, density_b200_table_init / _fold,
 * density_b200_cl_table_init / _fold and every density_b200_encode_sharded* driver takes its pointers by one rule: d_in and d_prev_quad
 * 4-byte aligned; d_out 2-byte aligned; every table, carry, transfer, word and flag buffer 4-byte aligned; d_out_size and d_total_size
 * 8-byte and d_seam8 4-byte aligned. A shard that does not end the stream is a multiple of 256 bytes. d_in and d_out may be NULL only
 * when their length is 0 (phase 2 of a Chameleon shard also takes a NULL d_out), d_flags and d_total_size may be NULL, an optional
 * table only where the entry says so. A misaligned or a missing pointer, or a phase called out of order, returns DENSITY_B200_EARG and
 * enqueues nothing; the drivers check every argument before their first collective.
 */

/*
 * Sharded Chameleon encode (one bit-exact stream cut across several GPUs / calls; SURVEY §8e).
 * The stream is cut at multiples of 256 bytes. Every shard runs phase 1 independently, the
 * 256 KiB last-writer tables are exchanged by the caller (torch.distributed all_gather in
 * density_b200/sharded.py), and phase 2 finishes the shard given the dictionary carried in
 * from all earlier shards. The concatenation of the shard outputs equals the output of one
 * chameleon_encode call over the concatenated input, provided the protection automaton stays
 * quiet (reported through *d_flags bit 0 otherwise; the caller then falls back to one device).
 */
typedef struct density_b200_shard density_b200_shard; /* opaque */
DENSITY_B200_API density_b200_shard* density_b200_shard_create(void);
DENSITY_B200_API void density_b200_shard_destroy(density_b200_shard*);
/* phase 1: flags with unknown carry-in; exports this shard's last-writer table (65536 x u32:
   bit 16 = bucket touched, low 16 bits = fingerprint) to d_table_out. */
DENSITY_B200_API int density_b200_shard_phase1(density_b200_shard*, const uint8_t* d_in, size_t n, int is_last_shard,
                              uint32_t* d_table_out, void* stream);
/* phase 2: d_carry_in = table state before this shard (65536 x u32, same encoding; for the first
   shard pass NULL). Writes the shard's piece of the stream to d_out and its size to *d_out_size. */
DENSITY_B200_API int density_b200_shard_phase2(density_b200_shard*, const uint32_t* d_carry_in, uint8_t* d_out, size_t cap,
                              uint64_t* d_out_size, uint32_t* d_flags, void* stream);
/* Fold shard tables left to right: d_acc = (d_next touched) ? d_next : d_acc, elementwise, 65536 entries.
   d_acc == NULL-initialised state is produced by density_b200_table_init. */
DENSITY_B200_API int density_b200_table_init(uint32_t* d_table, void* stream);
DENSITY_B200_API int density_b200_table_fold(uint32_t* d_acc, const uint32_t* d_next, void* stream);

/*
 * The same in C++ end to end (what bench.py --gpus N runs): one process per GPU, the exchange over NCCL (NVLink / NVSwitch).
 *   density_b200_sharded_unique_id   rank 0 makes the 128-byte NCCL id; the caller hands it to every rank (e.g. torch.distributed broadcast)
 *   density_b200_sharded_create      joins the communicator (world == 1: no NCCL needed, id may be NULL)
 *   density_b200_encode_sharded      phase 1 -> ncclAllGather of the 256 KiB tables -> ONE fold kernel -> phase 2 -> seam verdict
 *                                    (ncclAllGather of 32 bytes per rank: first / last block incompressible, quiet, size) -> optional
 *                                    variable-length gather of the pieces to `gather_root` (grouped ncclSend / ncclRecv at prefix-sum
 *                                    offsets). *d_flags != 0: the stream is not quiet (a copy-mode block somewhere, or two incompressible
 *                                    blocks across a cut): the pieces are void and the caller encodes on one device instead, or
 *                                    with density_b200_encode_sharded_protected below, which accepts such input.
 *                                    *d_total_size = length of the whole stream, on every rank. gather_root < 0: no gather, nothing blocks.
 *                                    d_gather NULL on the root: DENSITY_B200_EARG before any collective. The root's gather_cap reaches
 *                                    every rank with the seam words: when it is below the stream length every rank returns
 *                                    DENSITY_B200_ECAPACITY and no piece is sent.
 */
typedef struct density_b200_sharded density_b200_sharded; /* opaque */
DENSITY_B200_API int density_b200_sharded_unique_id(uint8_t* out128);
DENSITY_B200_API density_b200_sharded* density_b200_sharded_create(const uint8_t* nccl_unique_id_128, int rank, int world);
DENSITY_B200_API void density_b200_sharded_destroy(density_b200_sharded*);
DENSITY_B200_API int density_b200_encode_sharded(density_b200_sharded*, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                uint32_t* d_flags, uint64_t* d_total_size, int gather_root, uint8_t* d_gather, size_t gather_cap, void* stream);
/* stage times (ms) of the last encode_sharded or encode_sharded_cl call. Chameleon: [0] flag pass, [1] table exchange + fold, [2] carry /
   resolve / sizes / scan, [3] emit, [4] seams + gather. Cheetah / Lion: [0] phase 1, [1] P exchange + fold, [2] phase 2 + C exchange +
   fold, [3] phase 3, [4] seams + gather. encode_sharded_protected and encode_sharded_cl_protected: [0] phase 1, [1] the first table
   exchange + fold, [2] the rounds, sizes and scan, [3] emit, [4] seams + gather. */
DENSITY_B200_API int density_b200_sharded_profile(density_b200_sharded*, float* out_ms5);

/*
 * Sharded Chameleon encode with copy mode (DESIGN.md section 5): the quiet-only paths above refuse any input on which the protection
 * automaton fires (two incompressible blocks in a row anywhere: 512 bytes of compressed or random data). This path accepts it. The copy
 * map is the fixed point the single-device encoder iterates (flags under the map -> incompressible bits -> automaton -> new map); here
 * every round runs on all shards at once, with the dictionary and the automaton state carried over the cuts, so the shards compute the
 * single-device sequence of maps exactly. Shard r holds bytes [o_r, o_r + n_r) of one input, every non-final shard a multiple of 256
 * bytes; its first global block is o_r / 256. The concatenation of the pieces equals one chameleon_encode call over the whole input,
 * byte for byte, whenever the verdict is 0. Copy-mode blocks, penalties pending at a cut and incompressible pairs across a cut are all
 * accepted. The verdict is non-zero (the pieces are void; nothing is written past `cap`) only when the map did not settle within the
 * round budget, when the automaton's true path left the candidate states (penalty < 10, start 1..10: never seen on real data), or on an
 * error (capacity).
 *
 * Phase API on a density_b200_shard handle (any transport; W shards may run on one GPU). Per round k = 0, 1, ...:
 *   flags      k = 0: prot_phase1; k > 0: prot_next with a table. Exports the shard's last-writer table under the round's map.
 *   exchange   the tables of all shards; the carry-in of shard r is density_b200_table_init folded with the tables of shards < r.
 *   transfer   prot_transfer: DENSITY_B200_PROT_TRANSFER_WORDS u32, entry c = the automaton state at the shard end when the shard is
 *              entered in candidate state c (c = (previous_incompressible * 10 + start - 1) * 10 + penalty), or 0xFFFF.
 *   exchange   the transfers of all shards, in rank order.
 *   settle     prot_settle: the true incoming state (the transfers of shards < rank composed from c = 0, the stream start), the new
 *              copy map of the shard, and DENSITY_B200_PROT_ROUND_WORDS round words {blocks whose copy status changed, met 0xFFFF,
 *              settled before this round, 0}.
 *   exchange   the round words of all shards, in rank order; then prot_next: the global commit (settled when no shard changed and
 *              none met 0xFFFF: every later kernel returns at once), and with a table the next round's flags.
 * After the last round prot_next without a table commits it, and prot_finish emits. Every shard runs the same number of rounds; at
 * most density_b200_prot_round_budget() (prot_next with a table returns DENSITY_B200_EARG beyond it).
 */
#define DENSITY_B200_PROT_TRANSFER_WORDS 200
#define DENSITY_B200_PROT_ROUND_WORDS 4
#define DENSITY_B200_PROT_STATUS_WORDS 20
/* rounds of the iteration (16; density_b200_test_set_prot_rounds lowers it), of this path and of the Cheetah / Lion one
   (density_b200_cl_shard_prot_*, density_b200_encode_sharded_cl_protected) */
DENSITY_B200_API int density_b200_prot_round_budget(void);
/* round 0: flags with unknown carry-in, the last-writer table (as density_b200_shard_phase1) to d_table_out. d_in must stay valid and
   unchanged until prot_finish has been enqueued. */
DENSITY_B200_API int density_b200_shard_prot_phase1(density_b200_shard*, const uint8_t* d_in, size_t n, uint64_t first_block, int is_last_shard,
                                   uint32_t* d_table_out, void* stream);
/* d_carry_in: the dictionary before this shard under the round's map (NULL = stream start) */
DENSITY_B200_API int density_b200_shard_prot_transfer(density_b200_shard*, const uint32_t* d_carry_in, uint32_t* d_transfer_out, void* stream);
DENSITY_B200_API int density_b200_shard_prot_settle(density_b200_shard*, const uint32_t* d_all_transfers, int world, int rank,
                                   uint32_t* d_words_out, void* stream);
/* d_table_out NULL: commit the last round (then prot_finish) */
DENSITY_B200_API int density_b200_shard_prot_next(density_b200_shard*, const uint32_t* d_all_words, int world, uint32_t* d_table_out, void* stream);
/* sizes under the copy map, scan, emit: the piece to d_out, its size to *d_out_size (0 when refused) and 8 seam words to d_seam8 in the
   layout of density_b200_decode_shard_phase2 (words 0 and 1 are 0: incompressible blocks may meet at a cut; word 2 = refused or error).
   The verdict over all shards is cham_seam_verdict's rule: non-zero when any word 2 is set. */
DENSITY_B200_API int density_b200_shard_prot_finish(density_b200_shard*, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8,
                                   void* stream);
/* after the last commit (waits for the device): out[0] rounds until the map settled (0: not settled), [1] settled, [2] the incoming state
   of the last round run, penalty | start << 8 | previous_incompressible << 16 (~0: left the candidates), [3] met 0xFFFF, [4 + k] this
   shard's blocks whose copy status changed in round k (k < 16) */
DENSITY_B200_API int density_b200_shard_prot_status(density_b200_shard*, uint32_t* out20);
/* End to end over NCCL on a density_b200_sharded handle, with the arguments and gather semantics of density_b200_encode_sharded: an
   ncclAllGather of the shard lengths (the first global block) -> phase 1 -> the round budget of {ncclAllGather(tables) -> fold kernel ->
   transfer -> ncclAllGather(transfers, 800 bytes per rank) -> settle -> ncclAllGather(round words, 16 bytes) -> commit} -> finish ->
   seam verdict -> optional gather. Uses its own shard state in the handle; nothing blocks unless gather_root >= 0. */
DENSITY_B200_API int density_b200_encode_sharded_protected(density_b200_sharded*, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                          uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, int gather_root,
                                          uint8_t* d_gather, size_t gather_cap, void* stream);

/*
 * Sharded Cheetah / Lion encode (one bit-exact stream cut across several GPUs / calls; DESIGN.md section 5). Shard r holds bytes
 * [o_r, o_r + n_r) of one input; every non-final shard is a multiple of 256 bytes. The concatenation of the shard outputs equals one
 * cheetah_encode / lion_encode call over the whole input, byte for byte, whenever the verdict is 0. The verdict is non-zero (the pieces
 * are void and the caller encodes on one device) when the first shard's copy-map iteration did not settle; when the first shard is not
 * the last one and ends inside a copy run or with a copy penalty pending; when a later shard has two consecutive incompressible blocks
 * (it would need copy mode, which only the first shard may use); when a seam joins two incompressible blocks; or on an error (capacity).
 * The stream start belongs to the first shard: with that shard empty, the next one meets the cold-dictionary start without a copy map
 * and is normally refused.
 * Three phases around two table exchanges. Tables are stacks of u32 planes of 65536 entries (density_b200_cl_table_words u32 in all):
 *   P, Cheetah  {touched, last quad} per context
 *   P, Lion     {m, nu, l0..l4, v0..v4} per context: the shard's m local values, and the nu values of its undecided accesses, each of
 *               which removes one matching entry of the list carried into the shard
 *   C, both     {T, a, b} per bucket: T 0 untouched, 1 accessed with one value a, 2 ends as (a, b); 16-bit in-bucket fingerprints
 * A table describes what a shard does to the state carried into it; density_b200_cl_table_init gives the stream-start state and
 * density_b200_cl_table_fold(acc, next) makes acc "acc, then next", so the carry-in of shard r is init folded with the tables of
 * shards 0 .. r - 1 in order. All-zero tables are the identity (an empty shard).
 */
#define DENSITY_B200_CL_TABLE_P 0
#define DENSITY_B200_CL_TABLE_C 1
typedef struct density_b200_cl_shard density_b200_cl_shard; /* opaque */
/* alg: DENSITY_B200_CHEETAH or DENSITY_B200_LION (otherwise NULL, see density_b200_last_error) */
DENSITY_B200_API density_b200_cl_shard* density_b200_cl_shard_create(int alg);
DENSITY_B200_API void density_b200_cl_shard_destroy(density_b200_cl_shard*);
/* u32 words of one table of `kind` (DENSITY_B200_CL_TABLE_P / _C); 0 for a bad algorithm or kind */
DENSITY_B200_API size_t density_b200_cl_table_words(int alg, int kind);
/* phase 1: d_prev_quad: device pointer to the last quad (4 bytes) of the stream before this shard, NULL for the
   first shard, which alone runs the copy-map iteration (as the single-device encoder) and exports straight from its settled round.
   Exports the shard's P table. Phases 2 and 3 read d_in again: it must stay valid and unchanged until phase 3 has been enqueued. */
DENSITY_B200_API int density_b200_cl_shard_phase1(density_b200_cl_shard*, const uint8_t* d_in, size_t n, int is_last_shard,
                                 const uint32_t* d_prev_quad, uint32_t* d_table_p_out, void* stream);
/* phase 2: d_carry_p = the P state before this shard (NULL = stream start; the first shard ignores it). Exports the shard's C table. */
DENSITY_B200_API int density_b200_cl_shard_phase2(density_b200_cl_shard*, const uint32_t* d_carry_p, uint32_t* d_table_c_out, void* stream);
/* phase 3: d_carry_c = the C state before this shard (NULL = stream start; the first shard ignores it). Writes the shard's piece to d_out, its size
   to *d_out_size and its 8 seam words to d_seam8 in the layout of density_b200_decode_shard_phase2 ("last block incompressible" =
   previous_incompressible at the shard end; word 2 = this shard is refused). The verdict over all shards is that of the Chameleon
   sharded paths: non-zero when a word 2 is set or a seam joins two incompressible blocks. One phase 3 per phase 1. */
DENSITY_B200_API int density_b200_cl_shard_phase3(density_b200_cl_shard*, const uint32_t* d_carry_c, uint8_t* d_out, size_t cap,
                                 uint64_t* d_out_size, uint32_t* d_seam8, void* stream);
DENSITY_B200_API int density_b200_cl_table_init(int alg, int kind, uint32_t* d_table, void* stream);
DENSITY_B200_API int density_b200_cl_table_fold(int alg, int kind, uint32_t* d_acc, const uint32_t* d_next, void* stream);
/* End to end over NCCL on a density_b200_sharded handle, with the arguments and gather semantics of density_b200_encode_sharded:
   ncclAllGather of the last quads -> phase 1 -> ncclAllGather(P tables, 0.5 MiB per rank for Cheetah, 3 MiB for Lion) -> one fold
   kernel -> phase 2 -> ncclAllGather(C tables, 0.75 MiB) -> one fold kernel -> phase 3 -> seam words -> verdict -> optional gather.
   Uses its own workspace in the handle. */
DENSITY_B200_API int density_b200_encode_sharded_cl(density_b200_sharded*, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                   uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, int gather_root, uint8_t* d_gather,
                                   size_t gather_cap, void* stream);

/*
 * Sharded Cheetah / Lion encode with copy mode (DESIGN.md section 5): the path above refuses copy-mode blocks after the first shard,
 * penalties pending at a cut, incompressible pairs across a cut and an empty first shard; this one accepts them. It runs the copy-map
 * fixed point of the single-device encoder (flags under the map -> incompressible bits -> automaton -> new map) on all shards at once,
 * with the prediction tables, the chunk map, the context chain and the automaton state carried over the cuts. Shard r holds bytes
 * [o_r, o_r + n_r) of one input, every non-final shard a multiple of 256 bytes; its first global block is o_r / 128 (Cheetah) or o_r / 64
 * (Lion). The shard with o_r == 0 and n_r > 0 holds the stream start: it runs the staged iteration of the single-device encoder to the end
 * in phase 1 (the map of a prefix does not depend on what follows it, so that map is final); the others start from the empty map. Every
 * round extends the prefix on which the map agrees with the single call's by at least one block, and a map that a round leaves unchanged
 * is the single call's. The concatenation of the pieces equals one cheetah_encode / lion_encode call over the whole input, byte for
 * byte, whenever the verdict is 0. The verdict is non-zero (the pieces are void; nothing is written past `cap`) only when the staged
 * iteration of the shard at the stream start did not settle, when the rounds did not settle within the budget, when the automaton's true
 * path left the candidate states, or on an error (capacity).
 *
 * Phase API on a density_b200_cl_shard handle (any transport; W shards may run on one GPU): prot_phase1, then per round k = 0, 1, ...:
 *   P          prot_p: the context of the shard's first encoded quad from the round words of all shards (phase 1's for k = 0, else the
 *              round before's), ctx0 and pass P under the round's map, the shard's P table.
 *   exchange   the P tables; the carry-in of shard r is density_b200_cl_table_init folded with the tables of shards < r.
 *   C          prot_c: fold P from the carry-in, pass C, the shard's C table.
 *   exchange   the C tables, folded as the P tables.
 *   transfer   prot_transfer: fold C from the carry-in, sizes and incompressible bits, DENSITY_B200_PROT_TRANSFER_WORDS u32 as
 *              density_b200_shard_prot_transfer's.
 *   exchange   the transfers of all shards, in rank order.
 *   settle     prot_settle: the true incoming state, the shard's next map and DENSITY_B200_CL_PROT_ROUND_WORDS round words {blocks whose
 *              copy status changed, met 0xFFFF, settled before this round, 0, has an encoded quad, the last encoded quad, 0, 0} under
 *              the next map (a copied block contributes no quad; a shard without one passes the earlier value on).
 *   exchange   the round words of all shards, in rank order; then prot_next: the global commit (settled when no shard changed and
 *              none met 0xFFFF: every later kernel returns at once).
 * After at least one round, prot_finish emits. Every shard runs the same number of rounds; at most density_b200_prot_round_budget()
 * (prot_p returns DENSITY_B200_EARG beyond it). Per round and rank that is the P table (0.5 MiB Cheetah, 3 MiB Lion), the C table
 * (0.75 MiB), 800 bytes of transfer and 32 bytes of round words. A quiet density_b200_cl_shard_phase1 on the handle closes the prot
 * phases; an offset that is not a multiple of 256 returns DENSITY_B200_EARG.
 */
#define DENSITY_B200_CL_PROT_ROUND_WORDS 8
/* phase 1: the shard at the stream start (offset 0, n > 0) runs the staged copy-map iteration; the others take the empty map. Writes
   the shard's round words for round 0 (words 4-5: has an encoded quad, the last one, under that map; the rest 0). d_in must stay valid
   and unchanged until prot_finish has been enqueued. */
DENSITY_B200_API int density_b200_cl_shard_prot_phase1(density_b200_cl_shard*, const uint8_t* d_in, size_t n, uint64_t offset, int is_last_shard,
                                      uint32_t* d_words_out, void* stream);
/* d_all_words: [world][DENSITY_B200_CL_PROT_ROUND_WORDS], the round words of all shards from phase 1 or the round before */
DENSITY_B200_API int density_b200_cl_shard_prot_p(density_b200_cl_shard*, const uint32_t* d_all_words, int world, int rank, uint32_t* d_table_p_out,
                                 void* stream);
/* d_carry_p / d_carry_c: the P / C state before this shard under the round's map (the stream-start state for the first shard) */
DENSITY_B200_API int density_b200_cl_shard_prot_c(density_b200_cl_shard*, const uint32_t* d_carry_p, uint32_t* d_table_c_out, void* stream);
DENSITY_B200_API int density_b200_cl_shard_prot_transfer(density_b200_cl_shard*, const uint32_t* d_carry_c, uint32_t* d_transfer_out, void* stream);
DENSITY_B200_API int density_b200_cl_shard_prot_settle(density_b200_cl_shard*, const uint32_t* d_all_transfers, int world, int rank,
                                      uint32_t* d_words_out, void* stream);
DENSITY_B200_API int density_b200_cl_shard_prot_next(density_b200_cl_shard*, const uint32_t* d_all_words, int world, void* stream);
/* sizes under the committed map, scan, emit: the piece to d_out, its size to *d_out_size (0 when refused) and 8 seam words in the layout
   of density_b200_shard_prot_finish's (words 0 and 1 are 0; word 2 = refused or error) */
DENSITY_B200_API int density_b200_cl_shard_prot_finish(density_b200_cl_shard*, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8,
                                      void* stream);
/* after a commit (waits for the device), DENSITY_B200_PROT_STATUS_WORDS u32: out[0] the staged iteration of the shard at the stream start
   settled (1 on the other shards), [1] rounds until the map settled (0: not settled), [2] the incoming state of the last round run,
   penalty | start << 8 | previous_incompressible << 16 (~0: left the candidates), [3] met 0xFFFF, [4 + k] this shard's blocks whose copy
   status changed in round k (k < 16) */
DENSITY_B200_API int density_b200_cl_shard_prot_status(density_b200_cl_shard*, uint32_t* out20);
/* End to end over NCCL on a density_b200_sharded handle, with the arguments and gather semantics of density_b200_encode_sharded_cl:
   ncclAllGather(shard lengths, 8 bytes per rank), which the call waits for (the offsets decide which shard runs the staged iteration)
   -> phase 1 -> ncclAllGather(round words, 32 bytes) -> the round budget of {P -> ncclAllGather(P tables) -> fold kernel -> C ->
   ncclAllGather(C tables) -> fold kernel -> transfer -> ncclAllGather(transfers, 800 bytes) -> settle -> ncclAllGather(round words,
   32 bytes) -> commit} -> finish -> ncclAllGather(seam words) -> verdict -> optional gather. Uses its own workspace in the handle. */
DENSITY_B200_API int density_b200_encode_sharded_cl_protected(density_b200_sharded*, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out,
                                             size_t cap, uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, int gather_root,
                                             uint8_t* d_gather, size_t gather_cap, void* stream);

/*
 * Sharded decode. Every entry of the phase APIs of a Chameleon, Cheetah or Lion piece below, and every density_b200_decode_sharded*
 * driver, takes its pointers by one rule: d_in 2-byte aligned; d_out and every table, transfer, carry, word and walk-state buffer
 * 4-byte aligned; d_out_size 8-byte and d_seam8 4-byte aligned. d_in and d_out may be NULL only when their length is 0, an optional
 * table only where the entry says so. A misaligned or a missing pointer, or a phase called out of order, returns DENSITY_B200_EARG and
 * enqueues nothing: there is no in-order fallback on these paths.
 */

/*
 * Sharded Chameleon decode: the inverse of the sharded encode. Piece r is what shard r of a sharded encode produced (rank r's
 * d_out[0 .. d_out_size)), or equally the slice of a single-call stream at the prefix sums of those sizes. Decoding piece r with the
 * dictionary carried in from pieces < r gives back shard r byte for byte, so the concatenation equals chameleon_decode of the whole
 * stream. Quiet streams only, as for encode: the verdict is non-zero when a piece holds a copy-mode block, a seam joins two
 * incompressible blocks, a non-final piece does not decode to whole 256-byte blocks, or a piece is malformed or its output exceeds
 * `cap`. The decoded pieces are then void and the caller decodes the gathered stream on one device. Nothing is written past `cap`.
 */
typedef struct density_b200_decode_shard density_b200_decode_shard; /* opaque */
DENSITY_B200_API density_b200_decode_shard* density_b200_decode_shard_create(void);
DENSITY_B200_API void density_b200_decode_shard_destroy(density_b200_decode_shard*);
/* phase 1: boundaries and writer pass; exports the piece's last-writer table (shard format, as density_b200_shard_phase1) to
   d_table_out, including the PLAIN quads of the tail. cap = output capacity (sizes the boundary layout). Ends any piece in progress on
   the shard, protected steps included. */
DENSITY_B200_API int density_b200_decode_shard_phase1(density_b200_decode_shard*, const uint8_t* d_in, size_t n, size_t cap, int is_last_shard,
                                     uint32_t* d_table_out, void* stream);
/* phase 2: d_carry_in = dictionary before this piece (the left fold of the earlier pieces' tables over density_b200_table_init's
   state; NULL = stream start). Decodes into d_out, writes the decoded size to *d_out_size and the piece's 8 seam words to d_seam8:
   {first block incompressible, last block incompressible, not quiet or error, has blocks, decoded size lo, hi, 0, 0}, the layout
   of the encoder's seam words. One phase 2 per phase 1. */
DENSITY_B200_API int density_b200_decode_shard_phase2(density_b200_decode_shard*, const uint32_t* d_carry_in, uint8_t* d_out,
                                     uint64_t* d_out_size, uint32_t* d_seam8, void* stream);
/* End to end over NCCL on the communicator of a density_b200_sharded handle: phase 1 -> ncclAllGather(tables) -> fold kernel -> phase 2
   -> ncclAllGather(seam words) -> seam verdict. *d_flags != 0: the pieces are void. *d_total_size = the original length, on every
   rank (may be NULL). Never blocks; each rank gets back the shard it started with, so there is no gather. Uses its own workspace in
   the handle: encode_sharded and decode_sharded may alternate on one handle. */
DENSITY_B200_API int density_b200_decode_sharded(density_b200_sharded*, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, void* stream);

/*
 * Sharded Chameleon decode of streams with copy-mode blocks (DESIGN.md section 5): the inverse of density_b200_encode_sharded_protected,
 * and of the slices of a single-call chameleon_encode stream at its pieces' prefix sums, whatever the data. A piece's block boundaries
 * depend on the protection automaton state it is entered in and on the counter phase (the penalty start halves on every 16th block of
 * the stream), so every piece first exports its TRANSFER: DENSITY_B200_DECODE_PROT_TRANSFER_WORDS u32, entry c for the decode candidate
 * c = phase * 200 + (previous_incompressible * 10 + start - 1) * 10 + penalty (penalty 0..9, start 1..10, phase = blocks before the
 * piece mod 16; candidate 0 is the stream start) = the candidate in which the boundary walk leaves the piece exactly on its end,
 * 0xFFFF when that state is not a candidate, 0xFFFE when the walk does not end on the cut (overshoots it, stops short of it, a
 * malformed block, or more distinct walks than the walk keeps). The final piece's transfer is never read (all 0xFFFE).
 *   transfer  boundary rows of the piece and its transfer; cap = output capacity (as density_b200_decode_shard_phase1)
 *   phase 1   the transfers of the pieces before `rank` (d_all_transfers: [world][DENSITY_B200_DECODE_PROT_TRANSFER_WORDS], may be NULL
 *             for rank 0) composed from candidate 0 give the incoming state; boundaries from it, writer pass, and the piece's table
 *             exported to d_table_out (copy-mode blocks do not enter it)
 *   phase 2   as density_b200_decode_shard_phase2, seam words in its layout: words 0 and 1 are 0 (incompressible blocks may meet at a
 *             cut), word 2 is set when the composition met 0xFFFF or 0xFFFE, the piece is malformed or its output exceeds cap, or a
 *             non-final piece does not decode to whole 256-byte blocks.
 * One transfer, phase 1 and phase 2 in this order per piece; otherwise DENSITY_B200_EARG. Nothing is written past cap.
 */
#define DENSITY_B200_DECODE_PROT_TRANSFER_WORDS 3200
DENSITY_B200_API int density_b200_decode_shard_prot_transfer(density_b200_decode_shard*, const uint8_t* d_in, size_t n, size_t cap, int is_last_shard,
                                            uint32_t* d_transfer_out, void* stream);
DENSITY_B200_API int density_b200_decode_shard_prot_phase1(density_b200_decode_shard*, const uint32_t* d_all_transfers, int world, int rank,
                                          uint32_t* d_table_out, void* stream);
DENSITY_B200_API int density_b200_decode_shard_prot_phase2(density_b200_decode_shard*, const uint32_t* d_carry_in, uint8_t* d_out,
                                          uint64_t* d_out_size, uint32_t* d_seam8, void* stream);
/* End to end over NCCL, the arguments and semantics of density_b200_decode_sharded for any stream: transfer -> ncclAllGather(transfers,
   12.5 KiB) -> phase 1 -> ncclAllGather(tables) -> fold kernel -> phase 2 -> ncclAllGather(seam words) -> seam verdict. Never blocks;
   uses its own workspace in the handle. */
DENSITY_B200_API int density_b200_decode_sharded_protected(density_b200_sharded*, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                          uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, void* stream);

/*
 * Sharded Cheetah decode (DESIGN.md section 5). Piece r is what rank r of a sharded Cheetah encode produced (density_b200_cl_shard_phase3
 * or density_b200_encode_sharded_cl), or equally the slice of a single-call cheetah_encode stream at the prefix sums of those sizes.
 * Decoding every piece gives back its shard byte for byte whenever the verdict is 0, so the concatenation equals cheetah_decode of the
 * whole stream. The verdict is non-zero (the pieces are void and the caller decodes the gathered stream on one device) when:
 *   - the first piece, not being the last, ends inside a copy run or with a copy penalty pending;
 *   - a later piece is not quiet (a copy-mode block, two consecutive incompressible blocks) or a seam joins two incompressible blocks;
 *   - a non-final piece's blocks do not end exactly at its last byte, or meet copy mode there;
 *   - the prediction rounds did not settle within the round budget (density_b200_cheetah_decode_round_budget);
 *   - a piece is malformed, its output exceeds `cap`, or a non-final piece does not decode to whole 128-byte blocks.
 * Only the first piece may use copy mode: it holds the stream start, where every Cheetah stream has copy-mode blocks. Lion streams
 * (density_b200_decode_sharded_lion) and streams without known cuts are not decoded this way (density_b200_decode_sharded_cheetah_stream locates their pieces first).
 * Nothing is written past `cap`.
 *
 * Phase API of one piece (any transport; W pieces may run on one GPU): phase 1 -> exchange of the chunk-map transfers -> phase 2 -> rounds
 * (round_walk -> exchange of the prediction transfers and the round words -> round_fold), as many as the round budget -> phase 3 -> seam
 * words -> verdict (the rule of density_b200_decode_shard_phase2's words). Every piece runs the same number of rounds.
 * Tables are stacks of u32 planes of 65536 entries:
 *   chunk map (density_b200_cheetah_cmap_words() u32)  {tags, a, b} per bucket: slot s of the list the piece leaves is the literal in
 *                                                      plane 1 + s (tag bits 3s..3s+2 = 0) or slot t - 1 of the list carried in (tag t)
 *   predictions (density_b200_cl_table_words(DENSITY_B200_CHEETAH, DENSITY_B200_CL_TABLE_P) u32)  {touched, last value} per context: the
 *                                                      format of the Cheetah encoder's P table; fold it with density_b200_cl_table_init /
 *                                                      _fold(DENSITY_B200_CHEETAH, DENSITY_B200_CL_TABLE_P)
 *   round words (4 u32 per piece)                      {has an exit context, exit context, runs walked this round, an unknown was met}
 * The carry-in of piece r is the stream-start state (density_b200_cheetah_cmap_init, density_b200_cl_table_init) folded with the tables
 * of pieces 0 .. r - 1 in order; the round words are gathered from all pieces in rank order.
 */
typedef struct density_b200_cheetah_decode_shard density_b200_cheetah_decode_shard; /* opaque */
DENSITY_B200_API density_b200_cheetah_decode_shard* density_b200_cheetah_decode_shard_create(void);
DENSITY_B200_API void density_b200_cheetah_decode_shard_destroy(density_b200_cheetah_decode_shard*);
/* rounds every piece runs (40; density_b200_test_set_decode_rounds lowers it) */
DENSITY_B200_API int density_b200_cheetah_decode_round_budget(void);
/* u32 words of a chunk-map table (3 x 65536) */
DENSITY_B200_API size_t density_b200_cheetah_cmap_words(void);
/* phase 1: boundaries (the first piece from the fresh protection automaton, copy mode allowed), the end of the piece, unpack (literals and
   copy-mode blocks go to d_out at once), the symbolic chunk-map walk, and the piece's chunk-map transfer to d_cmap_out (may be NULL: no
   export). is_first: the piece holds the stream start; is_last: no stream byte follows it. d_in and d_out must stay valid until phase 3.
   Ends any piece in progress on the shard, protected steps included. */
DENSITY_B200_API int density_b200_cheetah_decode_shard_phase1(density_b200_cheetah_decode_shard*, const uint8_t* d_in, size_t n, uint8_t* d_out,
                                             size_t cap, int is_first, int is_last, uint32_t* d_cmap_out, void* stream);
/* phase 2: d_cmap_carry = the chunk map before this piece (NULL = stream start). Resolves the chunk-map reads, initialises the contexts. */
DENSITY_B200_API int density_b200_cheetah_decode_shard_phase2(density_b200_cheetah_decode_shard*, const uint32_t* d_cmap_carry, void* stream);
/* one round, first half: walks the runs that need it, exports this round's prediction transfer (d_pred_out, may be NULL) and the piece's 4
   round words (d_words4). DENSITY_B200_EARG once the round budget is used up. */
DENSITY_B200_API int density_b200_cheetah_decode_shard_round_walk(density_b200_cheetah_decode_shard*, uint32_t* d_pred_out, uint32_t* d_words4, void* stream);
/* second half: d_pred_carry = this round's prediction table before the piece (NULL = stream start), d_all_words = the round words of all
   `world` pieces in rank order, this piece being `rank`. Once no piece walked a run in a round, the rounds have settled and the kernels of
   the later rounds return at once. */
DENSITY_B200_API int density_b200_cheetah_decode_shard_round_fold(density_b200_cheetah_decode_shard*, const uint32_t* d_pred_carry,
                                                 const uint32_t* d_all_words, int world, int rank, void* stream);
/* phase 3: the tail of the final piece, the decoded size to *d_out_size (0 when the piece is refused) and the 8 seam words to d_seam8:
   {first block incompressible, previous_incompressible at the end, refused, has blocks, size lo, size hi, 0, 0}. */
DENSITY_B200_API int density_b200_cheetah_decode_shard_phase3(density_b200_cheetah_decode_shard*, uint64_t* d_out_size, uint32_t* d_seam8, void* stream);
/* Diagnostic, after phase 3 (synchronises the device): out4 = {rounds until settled, settled, run walks after round 0, rounds run}. */
DENSITY_B200_API int density_b200_cheetah_decode_shard_status(density_b200_cheetah_decode_shard*, uint32_t* out4);
/* the stream-start chunk map ((0, 0) in every bucket), and d_acc <- d_acc, then d_next */
DENSITY_B200_API int density_b200_cheetah_cmap_init(uint32_t* d_table, void* stream);
DENSITY_B200_API int density_b200_cheetah_cmap_fold(uint32_t* d_acc, const uint32_t* d_next, void* stream);
/* End to end over NCCL on a density_b200_sharded handle, with the arguments and semantics of density_b200_decode_sharded: phase 1 ->
   ncclAllGather(chunk-map transfers, 0.75 MiB per rank) -> one fold kernel -> phase 2 -> per round ncclAllGather(prediction transfers,
   0.5 MiB per rank) + ncclAllGather(round words) -> one fold kernel -> round fold, for every round of the budget -> phase 3 ->
   ncclAllGather(seam words) -> verdict. Never blocks, has no gather, uses its own workspace in the handle. */
DENSITY_B200_API int density_b200_decode_sharded_cheetah(density_b200_sharded*, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                        uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, void* stream);

/*
 * Sharded Cheetah decode of streams with copy-mode blocks (DESIGN.md section 5): the inverse of density_b200_encode_sharded_cl_protected
 * (Cheetah), and of the slices of a single-call cheetah_encode stream at its pieces' prefix sums, whatever the data. Copy mode, a pending
 * penalty, a cut inside a copy run and incompressible blocks on both sides of a cut are all accepted. As for Chameleon
 * (density_b200_decode_shard_prot_transfer), every piece first exports its TRANSFER, DENSITY_B200_DECODE_PROT_TRANSFER_WORDS u32 in the
 * same candidate encoding with the same 0xFFFF / 0xFFFE meaning; the final piece's is all 0xFFFE, an empty piece's the identity.
 *   prot_transfer  boundary rows of the piece and its transfer; the arguments of density_b200_cheetah_decode_shard_phase1 otherwise
 *   prot_phase1    the transfers of the pieces before `rank` (d_all_transfers: [world][DENSITY_B200_DECODE_PROT_TRANSFER_WORDS], may be
 *                  NULL for rank 0) composed from candidate 0 give the incoming state; then what density_b200_cheetah_decode_shard_phase1
 *                  does, from that state, with the chunk-map transfer to d_cmap_out (may be NULL)
 * The piece then runs phase 2, the rounds and phase 3 of the quiet path unchanged. Its phase 3 writes the seam words in their layout, with
 * words 0 and 1 = 0 and word 2 set when the composition met 0xFFFF or 0xFFFE, the piece is malformed or its output exceeds cap, the
 * rounds did not settle, the tail reported an error, or a non-final piece does not decode to whole 128-byte blocks. prot_transfer ->
 * prot_phase1 -> phase 2 -> rounds -> phase 3 in this order per piece (a quiet phase 1 in between closes the protected sequence);
 * otherwise DENSITY_B200_EARG. Nothing is written past cap.
 */
DENSITY_B200_API int density_b200_cheetah_decode_shard_prot_transfer(density_b200_cheetah_decode_shard*, const uint8_t* d_in, size_t n,
                                                    uint8_t* d_out, size_t cap, int is_first, int is_last, uint32_t* d_transfer_out,
                                                    void* stream);
DENSITY_B200_API int density_b200_cheetah_decode_shard_prot_phase1(density_b200_cheetah_decode_shard*, const uint32_t* d_all_transfers, int world,
                                                  int rank, uint32_t* d_cmap_out, void* stream);
/* End to end over NCCL, the arguments and semantics of density_b200_decode_sharded_cheetah for any stream: prot_transfer ->
   ncclAllGather(transfers, 12.5 KiB per rank) -> prot_phase1 -> the rest of density_b200_decode_sharded_cheetah. Never blocks; uses its
   own workspace in the handle. */
DENSITY_B200_API int density_b200_decode_sharded_cheetah_protected(density_b200_sharded*, const uint8_t* d_in, size_t n, uint8_t* d_out,
                                                  size_t cap, uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, void* stream);

/*
 * Sharded Lion decode (DESIGN.md section 5): the inverse of density_b200_encode_sharded_cl (Lion), and with the prot_* first step of
 * density_b200_encode_sharded_cl_protected (Lion), and of the slices of a single-call lion_encode stream at their pieces' prefix sums.
 * Boundaries, unpack and the chunk map run on every piece at once, as for Cheetah (Lion's chunk map is Cheetah's). The prediction walk
 * cannot: each piece's walk starts from the lists and the context the walk of the piece before it left, so the pieces walk one after the
 * other and a sharded Lion decode takes about as long as decoding the whole stream on one device. Decoding every piece gives back its
 * shard byte for byte whenever the verdict is 0. The quiet path refuses what Cheetah's refuses (copy mode or two consecutive
 * incompressible blocks in a later piece, a cut inside a copy run or with a penalty pending, incompressible blocks on both sides of a cut,
 * a non-final piece whose blocks do not end at its last byte); the protected path accepts all of these, with the transfers of
 * density_b200_cheetah_decode_shard_prot_transfer. Nothing is written past `cap`.
 *
 * Phase API of one piece (any transport; W pieces may run on one GPU), in this order per piece: phase 1 (or prot_transfer -> exchange
 * of the transfers -> prot_phase1) -> exchange of the chunk-map transfers -> phase 2 -> walk -> phase 3 -> seam words -> verdict (the
 * rule of density_b200_decode_shard_phase2's words).
 *   chunk map     the format of density_b200_cheetah_cmap_words, folded with density_b200_cheetah_cmap_init / _fold
 *   walk state    DENSITY_B200_LION_STATE_WORDS u32: the 65536 prediction lists (5 u32 each, context-major), then last_hash, then
 *                 padding. The state in front of the first piece is density_b200_lion_state_init's.
 */
#define DENSITY_B200_LION_STATE_WORDS (5 * 65536 + 8)
typedef struct density_b200_lion_decode_shard density_b200_lion_decode_shard; /* opaque */
DENSITY_B200_API density_b200_lion_decode_shard* density_b200_lion_decode_shard_create(void);
DENSITY_B200_API void density_b200_lion_decode_shard_destroy(density_b200_lion_decode_shard*);
/* phase 1: boundaries (the first piece from the fresh protection automaton, copy mode allowed), the end of the piece, unpack, the
   symbolic chunk-map walk and the piece's chunk-map transfer to d_cmap_out (may be NULL: no export). is_first: the piece holds the
   stream start; is_last: no stream byte follows it. d_in and d_out must stay valid until phase 3. Ends any piece in progress on the
   shard, protected steps included. */
DENSITY_B200_API int density_b200_lion_decode_shard_phase1(density_b200_lion_decode_shard*, const uint8_t* d_in, size_t n, uint8_t* d_out,
                                          size_t cap, int is_first, int is_last, uint32_t* d_cmap_out, void* stream);
/* phase 2: d_cmap_carry = the chunk map before this piece (NULL = stream start). Resolves the reads of carried-in chunk-map slots. */
DENSITY_B200_API int density_b200_lion_decode_shard_phase2(density_b200_lion_decode_shard*, const uint32_t* d_cmap_carry, void* stream);
/* the prediction walk: on entry d_state is the walk's state in front of the piece (the first piece starts from the stream-start state
   whatever it holds), on return the state behind it. An empty piece leaves it unchanged. */
DENSITY_B200_API int density_b200_lion_decode_shard_walk(density_b200_lion_decode_shard*, uint32_t* d_state, void* stream);
/* the stream-start walk state: zero lists, context 0 */
DENSITY_B200_API int density_b200_lion_state_init(uint32_t* d_state, void* stream);
/* phase 3: the tail of the final piece, the decoded size to *d_out_size (0 when the piece is refused) and the 8 seam words to d_seam8 in
   the layout of density_b200_cheetah_decode_shard_phase3 (non-final pieces decode to whole 64-byte blocks). */
DENSITY_B200_API int density_b200_lion_decode_shard_phase3(density_b200_lion_decode_shard*, uint64_t* d_out_size, uint32_t* d_seam8, void* stream);
/* the protected first step, with the arguments and semantics of density_b200_cheetah_decode_shard_prot_transfer / _prot_phase1 on the
   Lion geometry (35 entry offsets per 4 KiB chunk, the same 3200 candidates, 0xFFFF / 0xFFFE). Phase 2, the walk and phase 3 follow. */
DENSITY_B200_API int density_b200_lion_decode_shard_prot_transfer(density_b200_lion_decode_shard*, const uint8_t* d_in, size_t n, uint8_t* d_out,
                                                 size_t cap, int is_first, int is_last, uint32_t* d_transfer_out, void* stream);
DENSITY_B200_API int density_b200_lion_decode_shard_prot_phase1(density_b200_lion_decode_shard*, const uint32_t* d_all_transfers, int world,
                                               int rank, uint32_t* d_cmap_out, void* stream);
/* Diagnostic, after phase 3 (synchronises the device): the walk counts of this piece, the four values of density_b200_lion_decode_stats. */
DENSITY_B200_API int density_b200_lion_decode_shard_stats(density_b200_lion_decode_shard*, uint64_t* out4);
/* End to end over NCCL on a density_b200_sharded handle, with the arguments and semantics of density_b200_decode_sharded_cheetah: phase 1
   -> ncclAllGather(chunk-map transfers, 0.75 MiB per rank) -> one fold kernel -> phase 2 -> ncclRecv(walk state from rank - 1, on
   ranks > 0) -> walk -> ncclSend(walk state to rank + 1, on all but the last rank; 1.25 MiB) -> phase 3 -> ncclAllGather(seam words) ->
   verdict. The receive and the send are separate groups. Empty and refused pieces still receive and forward the state. Never blocks,
   has no gather, uses its own workspace in the handle. */
DENSITY_B200_API int density_b200_decode_sharded_lion(density_b200_sharded*, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                     uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, void* stream);
/* The same for any stream: prot_transfer -> ncclAllGather(transfers, 12.5 KiB per rank) -> prot_phase1 -> the rest of
   density_b200_decode_sharded_lion. */
DENSITY_B200_API int density_b200_decode_sharded_lion_protected(density_b200_sharded*, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                               uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, void* stream);

/*
 * Sharded decode of a stream whose cuts are not known: a stream written by one chameleon_encode call, by the reference library,
 * read from a file, or a gathered sharded stream without its piece sizes. The stream is cut at byte ranges; each rank finds
 * where its piece starts from the stream itself.
 *
 * Input layout. Rank r holds one contiguous device buffer (2-byte aligned): its RANGE, stream bytes [o_r, o_r + n_range_r), followed
 * by its HALO, the next n_halo_r = min(264, total - o_r - n_range_r) stream bytes (every byte a block starting inside the range can
 * reach). o_r is the sum of the n_range of the ranks before r; every non-last n_range is a multiple of 16384 (zero is allowed); the
 * last rank's n_range is any length and its halo is empty. Scattering a stream held by one rank is the caller's job.
 *
 * The range map (DENSITY_B200_LOCATE_MAP_WORDS u64): {n_range, n_halo}, then for each of the 132 possible even entry offsets e (2e
 * bytes into the range) {exit index x: the walk leaves the range at offset n_range + 2x and enters the next range at 2x; or ~0: the
 * walk reached the end of the stream; number of blocks it walked}.
 */
#define DENSITY_B200_LOCATE_MAP_WORDS 266
/* Enqueues the range map of d_in[0 .. n_range + n_halo) into d_map (device, 8-byte aligned). The scratch lives in the handle's
   workspace, which the next phase 1 overwrites, so the call ends any piece in progress on the shard, protected steps included. The layout is not checked here but by density_b200_locate_piece, which every rank
   runs on the same gathered maps. */
DENSITY_B200_API int density_b200_decode_locate(density_b200_decode_shard*, const uint8_t* d_in, size_t n_range, size_t n_halo,
                                uint64_t* d_map, void* stream);
/* Host only, needs no device. h_maps: the range maps of all `world` ranks in rank order. Checks the layout (non-last ranges multiples
   of 16384, each halo min(264, the bytes of the later ranges); DENSITY_B200_EARG otherwise, on every rank alike) and walks the maps
   from the stream start to `rank`. out4 = {start, end, blocks_before, is_final}: this rank's piece is d_in[start .. end), it begins
   after blocks_before blocks, and is_final = 1 when no stream byte follows it. A piece behind the end of the stream is empty. */
DENSITY_B200_API int density_b200_locate_piece(const uint64_t* h_maps, int world, int rank, uint64_t out4[4]);
/* End to end over NCCL on a density_b200_sharded handle: range map -> ncclAllGather(maps) -> one device-to-host copy and ONE host
   synchronisation (phase 1's launch grid depends on the piece length) -> density_b200_locate_piece -> the path of
   density_b200_decode_sharded on the located piece. *d_out_offset = where this piece's output starts in the original bytes;
   *d_flags, *d_total_size as density_b200_decode_sharded (d_out_offset and d_total_size may be NULL). Quiet streams only: a zero
   verdict proves every cut is a true block boundary (DESIGN.md section 5). For a quiet stream cap >= 2 * (n_range + n_halo) is always
   enough; a piece whose output does not fit is refused. Uses the handle's decode workspace. */
DENSITY_B200_API int density_b200_decode_sharded_stream(density_b200_sharded*, const uint8_t* d_in, size_t n_range, size_t n_halo,
                                       uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint64_t* d_out_offset,
                                       uint32_t* d_flags, uint64_t* d_total_size, void* stream);

/*
 * Sharded decode of a Cheetah stream whose cuts are not known (one cheetah_encode call, the reference library, a file, a gathered
 * sharded stream without its piece sizes), with the input layout of density_b200_decode_sharded_stream: range + halo of min(264, the
 * bytes of the later ranges), non-last ranges multiples of 16384 bytes. Each rank also passes its range_offset o_r (the sum of the
 * earlier n_range): the range with range_offset 0 and n_range > 0 holds the stream start.
 *
 * The range map (DENSITY_B200_CHEETAH_LOCATE_MAP_WORDS u64): {n_range, n_halo}, then for each of the 68 possible even entry offsets
 * {exit index or ~0, blocks} as in the Chameleon map (blocks taken as encoded blocks), then {range_offset, has_start_row, start exit,
 * start blocks}. Every Cheetah stream has copy-mode blocks near its start, which void the candidate walks there, so the range that
 * holds the stream start has a START ROW instead (its candidate rows are the identity): the exit and block count of the exact boundary
 * walk (codec.rs's main loop with the protection automaton, copy-mode blocks counted) from the stream start, the exit being the first
 * block start at or after n_range, or ~0 when the walk ends (fewer than 136 bytes left) in front of n_range.
 */
#define DENSITY_B200_CHEETAH_LOCATE_MAP_WORDS 142
/* Enqueues the range map of d_in[0 .. n_range + n_halo) into d_map (device, 8-byte aligned). Kernels: 4 on a range without the stream
   start (2 when it is empty), 11 on the range with it (the 9 boundary kernels of the exact walk, the identity rows, the start row).
   The scratch lives in the handle's workspace, which the next phase 1 overwrites, so the call ends any piece in progress on the shard,
   protected steps included; on the start range it holds one offset per 8 stream bytes. The layout is checked by density_b200_cheetah_locate_piece. */
DENSITY_B200_API int density_b200_cheetah_decode_locate(density_b200_cheetah_decode_shard*, const uint8_t* d_in, size_t n_range, size_t n_halo,
                                        uint64_t range_offset, uint64_t* d_map, void* stream);
/* Host only, needs no device. h_maps: the Cheetah range maps of all `world` ranks in rank order. Checks the layout as
   density_b200_locate_piece does, and that every range_offset is the sum of the earlier n_range and the start row is set on exactly
   the first non-empty range (DENSITY_B200_EARG otherwise, on every rank alike). Walks the maps from the start row: empty ranges pass
   the entry on, later ranges follow their candidate rows. out5 = {start, end, blocks_before, is_final, is_first}: this rank's piece is
   d_in[start .. end), it begins after blocks_before blocks, is_final = 1 when no stream byte follows it, is_first = 1 when it holds the
   stream start. A piece behind the end of the stream is empty. */
DENSITY_B200_API int density_b200_cheetah_locate_piece(const uint64_t* h_maps, int world, int rank, uint64_t out5[5]);
/* End to end over NCCL on a density_b200_sharded handle: Cheetah range map -> ncclAllGather(maps) -> one device-to-host copy and ONE
   host synchronisation -> density_b200_cheetah_locate_piece -> the path of density_b200_decode_sharded_cheetah on the located piece,
   with is_first / is_last of the located piece. *d_out_offset = where this piece's output starts in the original bytes; the other
   outputs as density_b200_decode_sharded_cheetah (d_out_offset and d_total_size may be NULL). Only the piece that holds the stream
   start may use copy mode; a zero verdict proves every cut is a true block boundary (DESIGN.md section 5). For a quiet piece
   cap >= 16 * (n_range + n_halo) is always enough; a piece whose output does not fit is refused, and nothing is written past cap. */
DENSITY_B200_API int density_b200_decode_sharded_cheetah_stream(density_b200_sharded*, const uint8_t* d_in, size_t n_range, size_t n_halo,
                                               uint64_t range_offset, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                               uint64_t* d_out_offset, uint32_t* d_flags, uint64_t* d_total_size, void* stream);

/*
 * Sharded decode of a stream whose cuts are not known, copy-mode blocks included (DESIGN.md section 5): archives, images, text mixed
 * with binary, Cheetah's cold start, whatever the data. The input layout of density_b200_decode_sharded_stream: range + halo of
 * min(264, the bytes of the later ranges), non-last ranges multiples of 16384 bytes; no range offset is needed.
 *
 * The PROTECTED RANGE MAP (u32): {n_range lo, n_range hi, n_halo lo, n_halo hi}, then for each entry offset e (2e bytes into the range;
 * 132 of them for Chameleon, 68 for Cheetah) and each decode candidate c (the encoding of density_b200_decode_shard_prot_transfer,
 * 3200 of them) one row at [4 + e * 3200 + c]: where the exact boundary walk (codec.rs's main loop with the protection automaton,
 * copy-mode blocks included) from offset 2e in candidate c leaves the range:
 *   exit | cand << 8  the first block start at or after n_range is n_range + 2 * exit (exit < 132 / 68), and the walk is in candidate
 *                     cand there;
 *   0xFF              the main loop ends (fewer than 264 / 136 bytes left) in front of n_range: the piece ends the stream;
 *   0xFFFF            the walk leaves the range in a state that is not a candidate;
 *   0xFFFE            more distinct walks than the walk keeps.
 * No row of the first two kinds equals 0xFFFF or 0xFFFE.
 */
#define DENSITY_B200_PROT_LOCATE_MAP_WORDS 422404
#define DENSITY_B200_CHEETAH_PROT_LOCATE_MAP_WORDS 217604
/* Enqueue the protected range map of d_in[0 .. n_range + n_halo) (2-byte aligned) into d_map (device, 4-byte aligned): the candidate
   rows of the quiet locate, then one head walk per entry offset (132 / 68 CTAs). The scratch lives in the shard's workspace, which the
   next phase 1 overwrites, so the call ends any piece in progress on the shard, protected steps included. The layout is checked by density_b200_prot_locate_piece. */
DENSITY_B200_API int density_b200_decode_prot_locate(density_b200_decode_shard*, const uint8_t* d_in, size_t n_range, size_t n_halo,
                                     uint32_t* d_map, void* stream);
DENSITY_B200_API int density_b200_cheetah_decode_prot_locate(density_b200_cheetah_decode_shard*, const uint8_t* d_in, size_t n_range,
                                             size_t n_halo, uint32_t* d_map, void* stream);
/* Host only, needs no device. alg: DENSITY_B200_CHAMELEON or DENSITY_B200_CHEETAH; h_maps: the protected range maps of all `world` ranks
   in rank order. Checks the layout as density_b200_locate_piece does (DENSITY_B200_EARG, on every rank alike, also for a malformed row on
   the path) and walks from entry 0, candidate 0 of the first non-empty range through every range; empty ranges pass the entry on.
   out6 = {start, end, is_final, is_first, entry candidate, refused}: this rank's piece is d_in[start .. end), entered in that candidate,
   is_final = 1 when no stream byte follows it, is_first = 1 when it holds the stream start. refused = 1 (all the others 0) when the walk
   met 0xFFFF or 0xFFFE anywhere, so every rank knows it. A piece behind the end of the stream is empty. */
DENSITY_B200_API int density_b200_prot_locate_piece(int alg, const uint32_t* h_maps, int world, int rank, uint64_t out6[6]);
/* Phase 1 of a located piece, from its entry candidate (< 3200) instead of composed transfers; the arguments of
   density_b200_decode_shard_prot_transfer otherwise. Followed by density_b200_decode_shard_prot_phase2, whose seam words it shares. */
DENSITY_B200_API int density_b200_decode_shard_prot_enter(density_b200_decode_shard*, const uint8_t* d_in, size_t n, size_t cap, int is_last_shard,
                                         uint32_t candidate, uint32_t* d_table_out, void* stream);
/* The same for Cheetah, the arguments of density_b200_cheetah_decode_shard_prot_phase1 with is_first / is_last of the located piece;
   followed by phase 2, the rounds and phase 3 unchanged. */
DENSITY_B200_API int density_b200_cheetah_decode_shard_prot_enter(density_b200_cheetah_decode_shard*, const uint8_t* d_in, size_t n,
                                                 uint8_t* d_out, size_t cap, int is_first, int is_last, uint32_t candidate,
                                                 uint32_t* d_cmap_out, void* stream);
/* End to end over NCCL on a density_b200_sharded handle, with the arguments of density_b200_decode_sharded_stream: protected range map ->
   ncclAllGather(maps, 1.6 MiB per rank) -> one compose kernel -> one device-to-host copy of 8 words and ONE host synchronisation ->
   prot_enter on the located piece -> ncclAllGather(tables) -> fold kernel -> prot_phase2 -> ncclAllGather(seam words) -> verdict. A
   refused composition is known on every rank from the same maps: each writes *d_flags = 1, *d_out_size = 0 (and 0 to d_out_offset and
   d_total_size when given) and enters no further collective. cap >= 2 * (n_range + n_halo) is always enough (a copy-mode block decodes to
   its own length); nothing is written past cap. Uses the handle's protected decode workspace. */
DENSITY_B200_API int density_b200_decode_sharded_stream_protected(density_b200_sharded*, const uint8_t* d_in, size_t n_range, size_t n_halo,
                                                 uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint64_t* d_out_offset,
                                                 uint32_t* d_flags, uint64_t* d_total_size, void* stream);
/* The same for a Cheetah stream (maps of 0.83 MiB per rank), then the path of density_b200_decode_sharded_cheetah on the located piece
   with its is_first / is_last: ncclAllGather(chunk-map transfers) -> fold -> phase 2 -> the rounds -> phase 3 -> ncclAllGather(seam
   words) -> verdict. cap >= 16 * (n_range + n_halo) is always enough. */
DENSITY_B200_API int density_b200_decode_sharded_cheetah_stream_protected(density_b200_sharded*, const uint8_t* d_in, size_t n_range,
                                                         size_t n_halo, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                                         uint64_t* d_out_offset, uint32_t* d_flags, uint64_t* d_total_size,
                                                         void* stream);

/*
 * A reused Codec INSTANCE (streaming continuation). In the reference `encode` / `decode` are methods of an instance
 * (/root/reference/src/codec/codec.rs:16,72,82) whose dictionary survives from call to call until clear_state()
 * (chameleon.rs:148-150, cheetah.rs:198-202, lion.rs:327-331), while the protection state is created inside every call
 * (codec.rs:75,85); the nine symbols above build a fresh instance per call (chameleon.rs:45-53). These mirror the instance:
 *   density_b200_codec_create(alg)  = X::new()        density_b200_codec_clear_state = Codec::clear_state
 *   density_b200_codec_encode       = Codec::encode   density_b200_codec_decode      = Codec::decode
 * Synchronous, host or device pointers, bytes written or 0 on error. Chameleon encode runs the run-parallel kernels with the
 * instance's dictionary carried in (buffers larger than HBM can be encoded piecewise, bit-exact with an instance on the CPU);
 * Cheetah / Lion and every decode run the exact in-order kernel on the instance's tables. An encode into a device output at
 * an odd address returns 0, as the nine encode symbols do (the encoders store 2-byte words).
 */
typedef struct density_b200_codec density_b200_codec; /* opaque */
DENSITY_B200_API density_b200_codec* density_b200_codec_create(int alg);
DENSITY_B200_API void density_b200_codec_destroy(density_b200_codec*);
DENSITY_B200_API int density_b200_codec_clear_state(density_b200_codec*);
DENSITY_B200_API size_t density_b200_codec_encode(density_b200_codec*, const uint8_t* input, size_t input_size, uint8_t* output, size_t output_size);
DENSITY_B200_API size_t density_b200_codec_decode(density_b200_codec*, const uint8_t* input, size_t input_size, uint8_t* output, size_t output_size);

/* ---- per-stage device timing of the last Chameleon encode on the current device ------- */
/* When enabled, density_b200_encode_device records CUDA events on the caller's stream around the flag pass
   and the emit pass of every call (ring of 64 calls; enable(1) resets it). density_b200_profile_get waits
   for them and returns the per-call AVERAGE over the recorded calls:
   out_ms[0] = flag pass, out_ms[1] = carry/resolve/sizes/scan, out_ms[2] = emit (milliseconds). */
DENSITY_B200_API void density_b200_profile_enable(int enable);
DENSITY_B200_API int density_b200_profile_get(float* out_ms);

/* ---- housekeeping ---------------------------------------------------------------------- */
/* Last error message of the calling thread's most recent failing call ("" if none). */
DENSITY_B200_API const char* density_b200_last_error(void);
/* Number of kernels this library has launched since load (for bench.py's gpu_launches). */
DENSITY_B200_API uint64_t density_b200_kernel_launches(void);
/* 1 if the last Chameleon encode on this device used the segment-parallel fast path end to end,
   0 if it had to fall back to the sequential protection-aware path. */
DENSITY_B200_API int density_b200_last_encode_was_fast(void);
/* Free all cached device workspaces. No other call may be in progress on any thread; the next call allocates them afresh. */
DENSITY_B200_API void density_b200_shutdown(void);
/* Test hook: cut every stage of the Cheetah / Lion copy-map iteration to k rounds (1..7, default 7) so that the host-resumed
   iteration of path 4 can be exercised on ordinary inputs. */
DENSITY_B200_API void density_b200_test_set_stage_rounds(int k);
/* Test hook: cut the round budget of the sharded Cheetah decode to k rounds (1..40, default 40) so that its "did not settle" refusal
   can be exercised. density_b200_decode_device does not read it. */
DENSITY_B200_API void density_b200_test_set_decode_rounds(int k);
/* Test hook: cut the round budget of the sharded copy-map iterations (density_b200_shard_prot_*, density_b200_encode_sharded_protected,
   density_b200_cl_shard_prot_*, density_b200_encode_sharded_cl_protected) to k rounds (1..16, default 16) so that their "did not
   settle" refusal can be exercised. The single-device encoders do not read it. */
DENSITY_B200_API void density_b200_test_set_prot_rounds(int k);
/* Test hook: resolve the NCCL entry points of the sharded drivers (ncclGetUniqueId, ncclCommInitRank, ncclCommDestroy, ncclAllGather,
   ncclSend, ncclRecv, ncclGroupStart, ncclGroupEnd, ncclGetErrorString) from the shared library at `path` instead of libnccl.so.2, e.g.
   a loopback library that serves several ranks in one process on one device; NULL restores the default lookup. DENSITY_B200_EARG when
   the library cannot be loaded, lacks one of the nine symbols, or while a density_b200_sharded handle with world > 1 is alive. Call it
   while no handle is being created. */
DENSITY_B200_API int density_b200_test_set_nccl_library(const char* path);
/* Diagnostic: the last copy-map iteration on the current device, per fixed-point round {first block whose copy status changed
   (~0: none), number of such blocks}: 16 rounds x 2 values. Synchronises the device. */
DENSITY_B200_API int density_b200_prot_debug(uint64_t* out32);
/* Library version string. */
DENSITY_B200_API const char* density_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* DENSITY_B200_H */
