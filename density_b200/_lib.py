"""ctypes binding of libdensity_b200.so (the C ABI declared in include/density_b200.h).

The library is the product; this module only loads it. It never falls back to a CPU implementation: if the
shared object is missing or CUDA is unusable the caller gets an exception / a 0 return, loudly.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("DENSITY_B200_SO") or os.path.join(_HERE, "libdensity_b200.so")  # env override: kernel-variant experiments

_c_u8p = ctypes.c_void_p
_SIGS = {
    # the reference's FFI surface: chameleon.rs:70-83, cheetah.rs:105-118, lion.rs:193-206
    **{f"{a}_{op}": (ctypes.c_size_t, [_c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t])
       for a in ("chameleon", "cheetah", "lion") for op in ("encode", "decode")},
    **{f"{a}_safe_encode_buffer_size": (ctypes.c_size_t, [ctypes.c_size_t]) for a in ("chameleon", "cheetah", "lion")},
    "density_b200_encode_device": (ctypes.c_int, [ctypes.c_int, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decode_device": (ctypes.c_int, [ctypes.c_int, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_encode_device_path": (ctypes.c_int, [ctypes.c_int, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]),
    "density_b200_decode_device_path": (ctypes.c_int, [ctypes.c_int, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]),
    "density_b200_decoded_size_device": (ctypes.c_int, [ctypes.c_int, _c_u8p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decoded_size": (ctypes.c_int, [ctypes.c_int, _c_u8p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_chameleon_decode_range_device": (ctypes.c_int, [_c_u8p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_uint64, _c_u8p,
                                                                   ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_chameleon_decode_range": (ctypes.c_int, [_c_u8p, ctypes.c_size_t, ctypes.c_uint64, _c_u8p, ctypes.c_uint64,
                                                            ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_chameleon_index_bytes": (ctypes.c_uint64, [ctypes.c_size_t, ctypes.c_uint64]),
    "density_b200_chameleon_index_build_device": (ctypes.c_int, [_c_u8p, ctypes.c_size_t, ctypes.c_uint64, _c_u8p, ctypes.c_size_t,
                                                                  ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_chameleon_index_build": (ctypes.c_int, [_c_u8p, ctypes.c_size_t, ctypes.c_uint64, _c_u8p, ctypes.c_size_t,
                                                           ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_chameleon_decode_range_indexed_device": (ctypes.c_int, [_c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_uint64,
                                                                           ctypes.c_uint64, _c_u8p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_chameleon_decode_range_indexed": (ctypes.c_int, [_c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_uint64, _c_u8p,
                                                                    ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_shard_create": (ctypes.c_void_p, []),
    "density_b200_shard_destroy": (None, [ctypes.c_void_p]),
    "density_b200_shard_phase1": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_shard_phase2": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_sharded_unique_id": (ctypes.c_int, [ctypes.c_void_p]),
    "density_b200_sharded_create": (ctypes.c_void_p, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]),
    "density_b200_sharded_destroy": (None, [ctypes.c_void_p]),
    "density_b200_encode_sharded": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p,
                                                   ctypes.c_void_p, ctypes.c_int, _c_u8p, ctypes.c_size_t, ctypes.c_void_p]),
    "density_b200_sharded_profile": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_float)]),
    "density_b200_prot_round_budget": (ctypes.c_int, []),
    "density_b200_shard_prot_phase1": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p,
                                                      ctypes.c_void_p]),
    "density_b200_shard_prot_transfer": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_shard_prot_settle": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_shard_prot_next": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_shard_prot_finish": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_shard_prot_status": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint32)]),
    "density_b200_encode_sharded_protected": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p,
                                                             ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, _c_u8p, ctypes.c_size_t,
                                                             ctypes.c_void_p]),
    "density_b200_decode_shard_create": (ctypes.c_void_p, []),
    "density_b200_decode_shard_destroy": (None, [ctypes.c_void_p]),
    "density_b200_decode_shard_phase1": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p,
                                                        ctypes.c_void_p]),
    "density_b200_decode_shard_phase2": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, _c_u8p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decode_shard_prot_transfer": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int,
                                                               ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decode_shard_prot_phase1": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                             ctypes.c_void_p]),
    "density_b200_decode_shard_prot_phase2": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, _c_u8p, ctypes.c_void_p, ctypes.c_void_p,
                                                             ctypes.c_void_p]),
    "density_b200_decode_sharded_protected": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p,
                                                             ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decode_sharded": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p,
                                                   ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decode_locate": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_locate_piece": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_decode_sharded_stream": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, _c_u8p, ctypes.c_size_t,
                                                          ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cl_shard_create": (ctypes.c_void_p, [ctypes.c_int]),
    "density_b200_cl_shard_destroy": (None, [ctypes.c_void_p]),
    "density_b200_cl_table_words": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int]),
    "density_b200_cl_shard_phase1": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                                    ctypes.c_void_p]),
    "density_b200_cl_shard_phase2": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cl_shard_phase3": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p,
                                                    ctypes.c_void_p]),
    "density_b200_cl_table_init": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cl_table_fold": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_encode_sharded_cl": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p,
                                                      ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, _c_u8p, ctypes.c_size_t, ctypes.c_void_p]),
    "density_b200_cl_shard_prot_phase1": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p,
                                                         ctypes.c_void_p]),
    "density_b200_cl_shard_prot_p": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cl_shard_prot_c": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cl_shard_prot_transfer": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cl_shard_prot_settle": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                         ctypes.c_void_p]),
    "density_b200_cl_shard_prot_next": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
    "density_b200_cl_shard_prot_finish": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p,
                                                         ctypes.c_void_p]),
    "density_b200_cl_shard_prot_status": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint32)]),
    "density_b200_encode_sharded_cl_protected": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t,
                                                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, _c_u8p,
                                                                ctypes.c_size_t, ctypes.c_void_p]),
    "density_b200_cheetah_decode_shard_create":(ctypes.c_void_p, []),
    "density_b200_cheetah_decode_shard_destroy": (None, [ctypes.c_void_p]),
    "density_b200_cheetah_decode_round_budget": (ctypes.c_int, []),
    "density_b200_cheetah_cmap_words": (ctypes.c_size_t, []),
    "density_b200_cheetah_decode_shard_phase1": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_int,
                                                                ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_decode_shard_phase2": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_decode_shard_round_walk": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_decode_shard_round_fold": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                                    ctypes.c_void_p]),
    "density_b200_cheetah_decode_shard_phase3": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_decode_shard_status": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint32)]),
    "density_b200_cheetah_cmap_init": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_cmap_fold": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decode_sharded_cheetah": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p,
                                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_decode_shard_prot_transfer": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t,
                                                                       ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_decode_shard_prot_phase1": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                                     ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decode_sharded_cheetah_protected": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t,
                                                                     ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_lion_decode_shard_create": (ctypes.c_void_p, []),
    "density_b200_lion_decode_shard_destroy": (None, [ctypes.c_void_p]),
    "density_b200_lion_decode_shard_phase1": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_int,
                                                             ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_lion_decode_shard_phase2": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_lion_decode_shard_walk": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_lion_state_init": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_lion_decode_shard_phase3": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_lion_decode_shard_prot_transfer": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t,
                                                                    ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_lion_decode_shard_prot_phase1": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                                  ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_lion_decode_shard_stats": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_decode_sharded_lion": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t, ctypes.c_void_p,
                                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decode_sharded_lion_protected": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t,
                                                                  ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_decode_locate": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint64,
                                                          ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_locate_piece": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_decode_sharded_cheetah_stream": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint64, _c_u8p,
                                                                  ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                                                  ctypes.c_void_p]),
    "density_b200_decode_prot_locate": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_decode_prot_locate": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p,
                                                               ctypes.c_void_p]),
    "density_b200_prot_locate_piece": (ctypes.c_int, [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_decode_shard_prot_enter": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int,
                                                            ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_cheetah_decode_shard_prot_enter": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t,
                                                                    ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decode_sharded_stream_protected": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, _c_u8p,
                                                                    ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                                                    ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_decode_sharded_cheetah_stream_protected": (ctypes.c_int, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, ctypes.c_size_t, _c_u8p,
                                                                            ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                                                            ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_codec_create": (ctypes.c_void_p, [ctypes.c_int]),
    "density_b200_codec_destroy": (None, [ctypes.c_void_p]),
    "density_b200_codec_clear_state": (ctypes.c_int, [ctypes.c_void_p]),
    "density_b200_codec_encode": (ctypes.c_size_t, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t]),
    "density_b200_codec_decode": (ctypes.c_size_t, [ctypes.c_void_p, _c_u8p, ctypes.c_size_t, _c_u8p, ctypes.c_size_t]),
    "density_b200_table_init": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_table_fold": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "density_b200_profile_enable": (None, [ctypes.c_int]),
    "density_b200_profile_get": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float)]),
    "density_b200_last_error": (ctypes.c_char_p, []),
    "density_b200_kernel_launches": (ctypes.c_uint64, []),
    "density_b200_last_encode_was_fast": (ctypes.c_int, []),
    "density_b200_decode_status": (ctypes.c_int, [ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_cheetah_decode_rounds": (ctypes.c_int, [ctypes.POINTER(ctypes.c_uint32)]),
    "density_b200_lion_decode_stats": (ctypes.c_int, [ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_encode_status": (ctypes.c_int, [ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_test_set_stage_rounds": (None, [ctypes.c_int]),
    "density_b200_test_set_decode_rounds": (None, [ctypes.c_int]),
    "density_b200_test_set_prot_rounds": (None, [ctypes.c_int]),
    "density_b200_test_set_nccl_library": (ctypes.c_int, [ctypes.c_char_p]),
    "density_b200_prot_debug": (ctypes.c_int, [ctypes.POINTER(ctypes.c_uint64)]),
    "density_b200_shutdown": (None, []),
    "density_b200_version": (ctypes.c_char_p, []),
}
EXPORTED_SYMBOLS = tuple(sorted(_SIGS))

_lib = None


class DensityB200Error(RuntimeError):
    pass


def load():
    """Load the CUDA library. Raises if it has not been built (python -m density_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise DensityB200Error(
                f"{SO_PATH} is missing: build it with `python -m density_b200.build` (nvcc, sm_90a). "
                "There is no CPU fallback.")
        L = ctypes.CDLL(SO_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)  # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def last_error():
    return load().density_b200_last_error().decode()
