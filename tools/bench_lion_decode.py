"""The parallel Lion decoder (density_b200_decode_device_path, path 0) against the in-order kernel (path 3) on one GPU.

    python tools/bench_lion_decode.py

  path0   1 GiB of synth_text, 256 MiB of synth_mixed and 256 MiB of noise, whole call (1 warm-up, 2 steps by default: a text call takes seconds)
  vs3     path 0 and path 3 on the first 64 MiB of each (path 3 runs at tens of MB/s: 1 warm-up on 1 MiB, 1 step)
  walk    the prediction walk kernel (ld_walk) alone, from torch.profiler in a separate run of one path-0 call per corpus, beside the
          whole call's time in that run
Each stream is encoded on the device (density_b200_encode_device); every timed output is compared with the input outside the timed
region. Rates are in uncompressed bytes. The GPU's name and power limit are read in the same run. One JSON line.
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
MIB = 1 << 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--text-bytes", type=int, default=1 << 30)
    ap.add_argument("--mixed-bytes", type=int, default=256 << 20)
    ap.add_argument("--prefix-bytes", type=int, default=64 << 20)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lion_decode needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import density_b200
    from density_b200 import synth
    lib = density_b200.load()
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    sz = torch.zeros(1, dtype=torch.int64, device=dev)
    name, power = gpu_name_and_power_limit()
    result, correct = {"metric": "lion_decode", "gpu": name, "power_limit": power}, True

    def encode(d_in):
        n = d_in.numel()
        d_enc = torch.empty(density_b200.Lion.safe_encode_buffer_size(n), dtype=torch.uint8, device=dev)
        assert lib.density_b200_encode_device(LION, d_in.data_ptr(), n, d_enc.data_ptr(), d_enc.numel(), sz.data_ptr(), stream()) == 0
        torch.cuda.synchronize()
        return d_enc[:int(sz.item())]

    def decoder(d_enc, d_out, path):
        return lambda: lib.density_b200_decode_device_path(LION, d_enc.data_ptr(), d_enc.numel(), d_out.data_ptr(), d_out.numel(), sz.data_ptr(),
                                                           stream(), path)

    def exact(d_out, d_in):
        torch.cuda.synchronize()
        return int(sz.item()) == d_in.numel() and bool(d_out.equal(d_in))

    inputs = [("text", synth.synth_text(args.text_bytes, device=dev)), ("mixed", synth.synth_mixed(args.mixed_bytes, device=dev)),
              ("noise", synth.random_bytes(args.mixed_bytes, 12345, device=dev))]
    for cname, d_in in inputs:
        n = d_in.numel()
        d_enc = encode(d_in)
        d_out = torch.empty(n, dtype=torch.uint8, device=dev)
        ms = timed(decoder(d_enc, d_out, 0), args.steps, args.warmup)
        ok = exact(d_out, d_in)
        correct &= ok
        st = (ctypes.c_uint64 * 4)()
        if lib.density_b200_lion_decode_stats(st) != 0:
            raise SystemExit("density_b200_lion_decode_stats failed: the timed decode did not run the parallel decoder")
        r = {"bytes": n, "stream_bytes": d_enc.numel(), "path0_ms": round(ms, 3), "path0_GBps": round(n / ms / 1e6, 3), "exact": ok,
             "quads": st[0], "predicted": st[1], "dependent_reads": st[2], "rows": st[3]}
        # the walk kernel's own time, from a profiled call of its own
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            decoder(d_enc, d_out, 0)()
            t1.record()
            torch.cuda.synchronize()
        walk_us = sum(e.device_time for e in prof.events() if "ld_walk" in e.name)
        r["profiled_call_ms"] = round(t0.elapsed_time(t1), 3)
        r["walk_kernel_ms"] = round(walk_us / 1e3, 3)
        # path 0 against path 3 on the same prefix
        p = min(args.prefix_bytes, n)
        d_pin = d_in[:p].clone()
        d_penc = encode(d_pin)
        d_pout = torch.empty(p, dtype=torch.uint8, device=dev)
        ms0 = timed(decoder(d_penc, d_pout, 0), args.steps, args.warmup)
        ok0 = exact(d_pout, d_pin)
        d_small = encode(d_pin[:MIB].clone())
        timed(decoder(d_small, torch.empty(MIB, dtype=torch.uint8, device=dev), 3), 1, 0)
        d_pout.zero_()
        ms3 = timed(decoder(d_penc, d_pout, 3), 1, 0)
        ok3 = exact(d_pout, d_pin)
        correct &= ok0 and ok3
        r.update({"prefix_bytes": p, "prefix_path0_ms": round(ms0, 3), "prefix_path3_ms": round(ms3, 3),
                  "prefix_path0_GBps": round(p / ms0 / 1e6, 3), "prefix_path3_GBps": round(p / ms3 / 1e6, 4),
                  "prefix_speedup": round(ms3 / ms0, 1), "prefix_exact": ok0 and ok3})
        result[cname] = r
        del d_in, d_enc, d_out, d_pin, d_penc, d_pout
    result["correct"] = correct
    print(json.dumps(result))


if __name__ == "__main__":
    main()
