"""Sharded decode of streams without known cuts that have copy-mode blocks (density_b200_decode_sharded_stream_protected and
density_b200_decode_sharded_cheetah_stream_protected) on one GPU, against the paths it extends.

    python tools/bench_sharded_stream_protected_decode.py [--baseline-lib OTHER/libdensity_b200.so]

For each algorithm (Chameleon, Cheetah) and each input (1 GiB of synth_text, 256 MiB of synth_mixed, 256 MiB of noise), encoded on the
device (density_b200_encode_device):
  locate          the protected range map of the whole stream as one range (density_b200_[cheetah_]decode_prot_locate: candidate rows,
                  then one head walk per entry offset, 132 / 68 CTAs)
  stream_prot     the driver at N = 1: locate, composition, one host synchronisation, prot_enter and the protected piece
  known_cut_prot  density_b200_decode_sharded[_cheetah]_protected of the same stream as one piece (its transfer walk, then the piece)
  decode_device   the single-device decoder
  transfer_walk   the known-cut transfer walk alone (density_b200_[cheetah_]decode_shard_prot_transfer of the stream as a non-final
                  piece); with --baseline-lib, the same call of another build of the library, alternated with it in this process
Every path is timed between CUDA events (warm-ups, then steps) and its output compared with the input outside the timed region. Rates
are in uncompressed bytes. The GPU's name and power limit are read in the same run. One JSON line.
"""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_sharded_decode import gpu_name_and_power_limit, timed  # noqa: E402

ALGS = {"chameleon": 0, "cheetah": 1}


def load_other(path):
    """another build of the library, for the transfer walk only"""
    from density_b200 import _lib
    L = ctypes.CDLL(os.path.abspath(path))
    for name in ("density_b200_decode_shard_create", "density_b200_decode_shard_prot_transfer", "density_b200_cheetah_decode_shard_create",
                 "density_b200_cheetah_decode_shard_prot_transfer"):
        fn = getattr(L, name)
        fn.restype, fn.argtypes = _lib._SIGS[name]
    return L


def transfer_walk(L, alg):
    """(shard, call(piece, d_out, n, transfer, stream)) of the known-cut transfer walk of library L"""
    if alg == "chameleon":
        h = L.density_b200_decode_shard_create()
        return lambda p, o, n, t, st: L.density_b200_decode_shard_prot_transfer(h, p.data_ptr(), p.numel(), n, 0, t.data_ptr(), st)
    h = L.density_b200_cheetah_decode_shard_create()
    return lambda p, o, n, t, st: L.density_b200_cheetah_decode_shard_prot_transfer(h, p.data_ptr(), p.numel(), o.data_ptr(), n, 1, 0,
                                                                                   t.data_ptr(), st)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--text-bytes", type=int, default=1 << 30)
    ap.add_argument("--mixed-bytes", type=int, default=256 << 20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--baseline-lib", default=None, help="another build of libdensity_b200.so: its known-cut transfer walk is timed too")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sharded_stream_protected_decode needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import density_b200
    from density_b200 import sharded, synth
    lib = density_b200.load()
    other = load_other(args.baseline_lib) if args.baseline_lib else None
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    dec = sharded.ShardedDecoder(dev)
    transfer = torch.empty(sharded.DECODE_PROT_TRANSFER_WORDS, dtype=torch.int32, device=dev)
    sz = torch.zeros(1, dtype=torch.int64, device=dev)
    fl = torch.ones(1, dtype=torch.int32, device=dev)
    result, correct = {"metric": "sharded_stream_protected_decode", "gpus": 1}, True
    inputs = [("text", lambda: synth.synth_text(args.text_bytes, device=dev)), ("mixed", lambda: synth.synth_mixed(args.mixed_bytes, device=dev)),
              ("noise", lambda: synth.random_bytes(args.mixed_bytes, 12345, device=dev))]
    for alg, aid in ALGS.items():
        walk = transfer_walk(lib, alg)
        walk_other = transfer_walk(other, alg) if other else None
        locate = lib.density_b200_decode_prot_locate if alg == "chameleon" else lib.density_b200_cheetah_decode_prot_locate
        loc_h = lib.density_b200_decode_shard_create() if alg == "chameleon" else lib.density_b200_cheetah_decode_shard_create()
        d_map = torch.empty(sharded.PROT_LOCATE_MAP_WORDS if alg == "chameleon" else sharded.CHEETAH_PROT_LOCATE_MAP_WORDS,
                            dtype=torch.int32, device=dev)
        codec = density_b200.CODECS[alg]
        for name, make in inputs:
            d_in = make()
            n = d_in.numel()
            d_enc = torch.empty(codec.safe_encode_buffer_size(n), dtype=torch.uint8, device=dev)
            rc = lib.density_b200_encode_device(aid, d_in.data_ptr(), n, d_enc.data_ptr(), d_enc.numel(), sz.data_ptr(), stream())
            torch.cuda.synchronize()
            if rc:
                raise SystemExit(f"encode_device rc={rc}: {density_b200._lib.last_error()}")
            piece = d_enc[:int(sz.item())]
            m = piece.numel()
            cap = n
            d_out = torch.empty(cap, dtype=torch.uint8, device=dev)
            out = {"bytes": n, "compressed_bytes": m}

            def check(ok_flags=True):
                return (not ok_flags or int(fl.item()) == 0) and int(sz.item()) == n and torch.equal(d_out[:n], d_in)

            ms = timed(lambda: locate(loc_h, piece.data_ptr(), m, 0, d_map.data_ptr(), stream()), args.steps, args.warmup)
            out["locate_ms"] = round(ms, 4)
            ms = timed(lambda: dec.decode_stream_protected(piece, m, d_out, sz, fl, alg=alg), args.steps, args.warmup)
            ok = check()
            out.update({"stream_prot_ms": round(ms, 4), "stream_prot_GBps": round(n / ms / 1e6, 2)})
            d_out.zero_()
            ms = timed(lambda: dec.decode_protected(piece, d_out, sz, fl, alg=alg), args.steps, args.warmup)
            ok &= check()
            out.update({"known_cut_prot_ms": round(ms, 4), "known_cut_prot_GBps": round(n / ms / 1e6, 2)})
            d_out.zero_()
            ms = timed(lambda: lib.density_b200_decode_device(aid, piece.data_ptr(), m, d_out.data_ptr(), cap, sz.data_ptr(), stream()),
                       args.steps, args.warmup)
            ok &= check(False)
            out.update({"decode_device_ms": round(ms, 4), "decode_device_GBps": round(n / ms / 1e6, 2)})
            walks = [("transfer_walk_ms", walk)] + ([("transfer_walk_baseline_ms", walk_other)] if walk_other else [])
            acc = {k: [] for k, _ in walks}
            for _ in range(3):                          # alternated, so that both builds see the same machine state
                for k, w in walks:
                    acc[k].append(timed(lambda: w(piece, d_out, cap, transfer, stream()), args.steps, args.warmup))
            out.update({k: round(sorted(v)[1], 4) for k, v in acc.items()})
            correct &= bool(ok)
            result[f"{alg}_{name}"] = out
            del d_in, d_enc, d_out, piece
            torch.cuda.empty_cache()
    name, power = gpu_name_and_power_limit()
    result.update({"correct": bool(correct), "gpu": name, "power_limit": power, "steps": args.steps, "warmup": args.warmup})
    print(json.dumps(result), flush=True)
    dec.close()
    if not correct:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
