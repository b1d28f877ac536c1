"""Time the Chameleon range decode (density_b200_chameleon_decode_range_device) of a 1 MiB window at the start, the middle and the end of a
stream, next to the decoded-size query (the range decode's locate step walks the same boundaries) and decode_device of the whole stream,
with CUDA events; and the device memory each call allocates.

Workloads: 1 GiB of synthetic text, 256 MiB of synth_mixed and of noise (copy-mode blocks), each encoded by the library. Times are the
mean of --reps calls after 3 warm-ups. Scratch: the device memory the library holds after one call from a released state
(density_b200_shutdown, then torch.cuda.mem_get_info around the call, the smaller of two tries), i.e. the workspace with its growth
slack; decode_device also needs the caller's output buffer of the full decoded size, reported as decode_output_bytes. Prints the card's name and power limit first, then
one JSON line per workload and window. Usage: python tools/bench_decode_range.py [--reps R]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import density_b200  # noqa: E402
from density_b200 import codec, synth  # noqa: E402

MIB, GIB = 1 << 20, 1 << 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def timed(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def scratch(lib, fn):
    """device bytes the library holds after one call from a released state (the smaller of two tries: the free-memory count of the
    device can move for reasons of its own)"""
    got = []
    for _ in range(2):
        torch.cuda.synchronize()
        lib.density_b200_shutdown()
        torch.cuda.empty_cache()
        free0 = torch.cuda.mem_get_info()[0]
        fn()
        torch.cuda.synchronize()
        got.append(free0 - torch.cuda.mem_get_info()[0])
    return min(got)


def workload(lib, kind, n, reps):
    data = {"text": lambda: synth.synth_text(n, device="cuda"), "mixed": lambda: synth.synth_mixed(n, device="cuda"),
            "noise": lambda: synth.random_bytes(n, 5, device="cuda")}[kind]()
    enc = torch.empty(density_b200.Chameleon.safe_encode_buffer_size(n), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    codec.encode_device("chameleon", data, enc, sz)
    torch.cuda.synchronize()
    m = int(sz.item())
    res = torch.zeros(3, dtype=torch.int64, device="cuda")
    win = torch.empty(MIB, dtype=torch.uint8, device="cuda")
    size_q = torch.zeros(2, dtype=torch.int64, device="cuda")
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    dec = lambda: codec.decode_device("chameleon", enc, m, out, sz)      # noqa: E731
    dec_scratch = scratch(lib, dec)
    d_ms = timed(dec, 1, reps)
    assert int(sz.item()) == n and torch.equal(out, data), f"{kind}: decode differs"
    del out
    torch.cuda.empty_cache()
    q_ms = timed(lambda: codec.decoded_size_device("chameleon", enc, m, size_q), 3, reps)
    rows = []
    for where, first in (("start", 0), ("middle", n // 2), ("end", n - MIB)):
        rng = lambda: codec.decode_range_device(enc, m, first, win, res)   # noqa: E731
        rng_scratch = scratch(lib, rng)
        r_ms = timed(rng, 3, reps)
        assert res.cpu().tolist() == [MIB, n, 0] and torch.equal(win, data[first:first + MIB]), f"{kind} {where}: window differs"
        rows.append({"corpus": kind, "input_bytes": n, "stream_bytes": m, "window": where, "first": first, "len": MIB,
                     "range_ms": round(r_ms, 3), "range_scratch_bytes": rng_scratch, "decoded_size_ms": round(q_ms, 3),
                     "decode_ms": round(d_ms, 3), "decode_scratch_bytes": dec_scratch, "decode_output_bytes": n,
                     "range_share_of_decode": round(r_ms / d_ms, 3)})
    del data, enc
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    lib = density_b200.load()
    print(json.dumps(card()), flush=True)
    for kind, n in (("text", GIB), ("mixed", 256 * MIB), ("noise", 256 * MIB)):
        for row in workload(lib, kind, n, args.reps):
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
