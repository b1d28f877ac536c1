"""Sharded Lion decode (density_b200_decode_sharded_lion and _protected) at N = 1 on one GPU, against decode_device.

    python tools/bench_sharded_lion_decode.py

  text / mixed / noise   256 MiB of synth_text, synth_mixed and noise: decode_sharded_lion and decode_sharded_lion_protected against
                         decode_device (the cost of the piece path around the same walk: the chunk-map export, the copies of the walk's
                         state in and out, and for the protected driver the transfer walk and the seeded boundaries)
  walk                   the transfer walk of each stream alone (density_b200_lion_decode_shard_prot_transfer of the whole stream as a
                         non-final piece: candidate rows + head walk over 4 KiB chunks), the cost a non-final protected piece pays
Each stream is encoded on the device (density_b200_encode_device), every path is timed between CUDA events and its output compared with
the input outside the timed region. The Lion walk runs at about 0.05 GB/s on text, so the defaults are 1 warm-up and 3 steps. Rates are
in uncompressed bytes. The GPU's name and power limit are read in the same run. One JSON line.
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

LION = 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=256 << 20)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sharded_lion_decode needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import density_b200
    from density_b200 import sharded, synth
    lib = density_b200.load()
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    dec = sharded.ShardedLionDecoder(dev)
    walker = lib.density_b200_lion_decode_shard_create()
    transfer = torch.empty(sharded.DECODE_PROT_TRANSFER_WORDS, dtype=torch.int32, device=dev)
    sz = torch.zeros(1, dtype=torch.int64, device=dev)
    fl = torch.ones(1, dtype=torch.int32, device=dev)
    result, correct = {"metric": "sharded_lion_decode", "gpus": 1}, True
    inputs = [("text", synth.synth_text(args.bytes, device=dev)), ("mixed", synth.synth_mixed(args.bytes, device=dev)),
              ("noise", synth.random_bytes(args.bytes, 12345, device=dev))]
    for name, d_in in inputs:
        n = d_in.numel()
        d_enc = torch.empty(density_b200.Lion.safe_encode_buffer_size(n), dtype=torch.uint8, device=dev)
        rc = lib.density_b200_encode_device(LION, d_in.data_ptr(), n, d_enc.data_ptr(), d_enc.numel(), sz.data_ptr(), stream())
        torch.cuda.synchronize()
        if rc:
            raise SystemExit(f"encode_device rc={rc}: {density_b200._lib.last_error()}")
        piece = d_enc[:int(sz.item())]
        d_out = torch.empty(n, dtype=torch.uint8, device=dev)
        row = {"bytes": n, "compressed_bytes": piece.numel()}
        paths = [("decode_device", lambda: lib.density_b200_decode_device(LION, piece.data_ptr(), piece.numel(), d_out.data_ptr(), n,
                                                                             sz.data_ptr(), stream()), False),
                 ("sharded", lambda: dec.decode(piece, d_out, sz, fl), True),
                 ("sharded_protected", lambda: dec.decode_protected(piece, d_out, sz, fl), True)]
        for label, fn, has_flags in paths:
            d_out.zero_()
            fl.fill_(1)
            ms = timed(fn, args.steps, args.warmup)
            ok = int(sz.item()) == n and torch.equal(d_out, d_in) and (not has_flags or int(fl.item()) == 0)
            correct &= ok
            row[f"{label}_ms"] = round(ms, 3)
            row[f"{label}_GBps"] = round(n / ms / 1e6, 4)
        base = row["decode_device_ms"]
        row["sharded_vs_decode_device_pct"] = round(100.0 * (row["sharded_ms"] / base - 1.0), 2)
        row["sharded_protected_vs_decode_device_pct"] = round(100.0 * (row["sharded_protected_ms"] / base - 1.0), 2)
        ms_walk = timed(lambda: lib.density_b200_lion_decode_shard_prot_transfer(walker, piece.data_ptr(), piece.numel(), d_out.data_ptr(),
                                                                                 n, 1, 0, transfer.data_ptr(), stream()),
                        args.steps, args.warmup)
        row["transfer_walk_ms"] = round(ms_walk, 4)
        row["transfer_walk_ns_per_byte"] = round(ms_walk * 1e6 / n, 4)
        result[name] = row
        del d_in, d_enc, d_out, piece
    name, power = gpu_name_and_power_limit()
    result.update({"correct": bool(correct), "gpu": name, "power_limit": power, "steps": args.steps, "warmup": args.warmup})
    print(json.dumps(result), flush=True)
    lib.density_b200_lion_decode_shard_destroy(walker)
    dec.close()
    if not correct:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
