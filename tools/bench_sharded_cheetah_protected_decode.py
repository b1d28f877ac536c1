"""Sharded Cheetah decode of streams with copy-mode blocks (density_b200_decode_sharded_cheetah_protected) on one GPU, against the paths
it extends.

    python tools/bench_sharded_cheetah_protected_decode.py

  text   1 GiB of synth_text: decode_sharded_cheetah_protected against decode_sharded_cheetah (quiet data: the cost of the extra exchange,
         the transfer walk and the seeded boundaries)
  mixed  256 MiB of synth_mixed and of noise: decode_sharded_cheetah_protected against decode_device (decode_sharded_cheetah refuses
         copy mode after the first piece)
  walk   the transfer walk of each stream alone (density_b200_cheetah_decode_shard_prot_transfer of the whole stream as a non-final piece:
         candidate rows + head walk over 4 KiB chunks)
Each stream is encoded on the device (density_b200_encode_device), every path is timed between CUDA events (3 warm-ups, 20 steps)
and its output compared with the input outside the timed region. Rates are in uncompressed bytes. The GPU's name and power limit are
read in the same run. One JSON line.
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

CHEETAH = 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--text-bytes", type=int, default=1 << 30)
    ap.add_argument("--mixed-bytes", type=int, default=256 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sharded_cheetah_protected_decode needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import density_b200
    from density_b200 import sharded, synth
    lib = density_b200.load()
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    dec = sharded.ShardedDecoder(dev)
    walker = lib.density_b200_cheetah_decode_shard_create()
    transfer = torch.empty(sharded.DECODE_PROT_TRANSFER_WORDS, dtype=torch.int32, device=dev)
    sz = torch.zeros(1, dtype=torch.int64, device=dev)
    fl = torch.ones(1, dtype=torch.int32, device=dev)
    result, correct = {"metric": "sharded_cheetah_protected_decode", "gpus": 1}, True
    inputs = [("text", synth.synth_text(args.text_bytes, device=dev), "decode_sharded_cheetah"),
              ("mixed", synth.synth_mixed(args.mixed_bytes, device=dev), "decode_device"),
              ("noise", synth.random_bytes(args.mixed_bytes, 12345, device=dev), "decode_device")]
    for name, d_in, other in inputs:
        n = d_in.numel()
        d_enc = torch.empty(density_b200.Cheetah.safe_encode_buffer_size(n), dtype=torch.uint8, device=dev)
        rc = lib.density_b200_encode_device(CHEETAH, d_in.data_ptr(), n, d_enc.data_ptr(), d_enc.numel(), sz.data_ptr(), stream())
        torch.cuda.synchronize()
        if rc:
            raise SystemExit(f"encode_device rc={rc}: {density_b200._lib.last_error()}")
        piece = d_enc[:int(sz.item())]
        d_out = torch.empty(n, dtype=torch.uint8, device=dev)
        ms = timed(lambda: dec.decode_protected(piece, d_out, sz, fl, alg="cheetah"), args.steps, args.warmup)
        ok = int(fl.item()) == 0 and int(sz.item()) == n and torch.equal(d_out, d_in)
        d_out.zero_()
        if other == "decode_sharded_cheetah":
            ms_other = timed(lambda: dec.decode(piece, d_out, sz, fl, alg="cheetah"), args.steps, args.warmup)
            ok_other = int(fl.item()) == 0 and int(sz.item()) == n and torch.equal(d_out, d_in)
        else:
            ms_other = timed(lambda: lib.density_b200_decode_device(CHEETAH, piece.data_ptr(), piece.numel(), d_out.data_ptr(), n,
                                                                    sz.data_ptr(), stream()), args.steps, args.warmup)
            ok_other = int(sz.item()) == n and torch.equal(d_out, d_in)
        ms_walk = timed(lambda: lib.density_b200_cheetah_decode_shard_prot_transfer(walker, piece.data_ptr(), piece.numel(), d_out.data_ptr(),
                                                                                    n, 1, 0, transfer.data_ptr(), stream()),
                        args.steps, args.warmup)
        correct &= ok and ok_other
        result[name] = {"bytes": n, "compressed_bytes": piece.numel(), "protected_ms": round(ms, 4),
                        "protected_GBps": round(n / ms / 1e6, 2), f"{other}_ms": round(ms_other, 4),
                        f"{other}_GBps": round(n / ms_other / 1e6, 2), "transfer_walk_ms": round(ms_walk, 4)}
        del d_in, d_enc, d_out, piece
    name, power = gpu_name_and_power_limit()
    result.update({"correct": bool(correct), "gpu": name, "power_limit": power, "steps": args.steps, "warmup": args.warmup})
    print(json.dumps(result), flush=True)
    lib.density_b200_cheetah_decode_shard_destroy(walker)
    dec.close()
    if not correct:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
