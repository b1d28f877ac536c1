"""Time the Chameleon seek index (density_b200_chameleon_index_build_device, density_b200_chameleon_decode_range_indexed_device) against the
non-indexed range decode and decode_device, with CUDA events.

Workloads: 1 GiB of synthetic text, 256 MiB of synth_mixed and of noise (copy-mode blocks), each encoded by the library. Per workload:
  - the build at intervals of 4, 16 and 64 MiB: time (mean of --reps builds after 1 warm-up; the build waits once on the host) and the
    index's size;
  - at the 16 MiB interval, a 1 MiB window at the start, the middle and the end: indexed, non-indexed, and decode_device of the whole
    stream (mean of --reps calls after 3 warm-ups);
  - 1000 random 4 KiB windows, indexed and non-indexed (the non-indexed run is cut to --random-plain reads and scaled, because each read
    walks the whole stream), host clock around the reads and a device synchronise; the first three reads are checked afterwards;
  - the synchronous indexed decode of a 1 MiB window from a pageable host copy of the stream and of the index.
Prints the card's name and power limit first, then one JSON line per measurement. Usage:
python tools/bench_chameleon_index.py [--reps R] [--random-plain K]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
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


def workload(lib, kind, n, reps, random_plain):
    data = {"text": lambda: synth.synth_text(n, device="cuda"), "mixed": lambda: synth.synth_mixed(n, device="cuda"),
            "noise": lambda: synth.random_bytes(n, 5, device="cuda")}[kind]()
    enc = torch.empty(density_b200.Chameleon.safe_encode_buffer_size(n), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    codec.encode_device("chameleon", data, enc, sz)
    torch.cuda.synchronize()
    m = int(sz.item())
    res = torch.zeros(3, dtype=torch.int64, device="cuda")
    base = {"corpus": kind, "input_bytes": n, "stream_bytes": m}
    rows = []
    indexes = {}
    for interval in (4 * MIB, 16 * MIB, 64 * MIB):
        idx = torch.empty(lib.density_b200_chameleon_index_bytes(m, interval), dtype=torch.uint8, device="cuda")
        b_ms = timed(lambda: codec.index_build_device(enc, m, interval, idx, res), 1, reps)
        size = int(res[0].item())
        assert res.cpu().tolist()[1:] == [n, 0], f"{kind}: build result {res.cpu().tolist()}"
        indexes[interval] = (idx, size)
        rows.append(dict(base, measure="build", interval=interval, build_ms=round(b_ms, 3), index_bytes=size,
                         checkpoints=int(idx[48:56].cpu().numpy().view(np.uint64)[0])))
    idx, ilen = indexes[16 * MIB]
    del indexes
    win = torch.empty(MIB, dtype=torch.uint8, device="cuda")
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_ms = timed(lambda: codec.decode_device("chameleon", enc, m, out, sz), 1, reps)
    assert int(sz.item()) == n and torch.equal(out, data), f"{kind}: decode differs"
    del out
    torch.cuda.empty_cache()
    for where, first in (("start", 0), ("middle", n // 2), ("end", n - MIB)):
        ix = lambda: codec.decode_range_indexed_device(enc, m, idx, ilen, first, win, res)   # noqa: E731
        i_ms = timed(ix, 3, reps)
        assert res.cpu().tolist() == [MIB, n, 0] and torch.equal(win, data[first:first + MIB]), f"{kind} {where}: indexed window differs"
        r_ms = timed(lambda: codec.decode_range_device(enc, m, first, win, res), 3, reps)
        assert res.cpu().tolist() == [MIB, n, 0] and torch.equal(win, data[first:first + MIB]), f"{kind} {where}: window differs"
        rows.append(dict(base, measure="window_1MiB", interval=16 * MIB, window=where, indexed_ms=round(i_ms, 3), range_ms=round(r_ms, 3),
                         decode_ms=round(d_ms, 3)))
    rng = np.random.default_rng(1)
    firsts = rng.integers(0, n - 4096, 1000)
    small = torch.empty(4096, dtype=torch.uint8, device="cuda")
    for name, fn, count in (("indexed", lambda f: codec.decode_range_indexed_device(enc, m, idx, ilen, f, small, res), 1000),
                            ("range", lambda f: codec.decode_range_device(enc, m, f, small, res), min(random_plain, 1000))):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for f in firsts[:count]:
            fn(int(f))
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        for f in firsts[:3]:
            fn(int(f))
            torch.cuda.synchronize()
            assert torch.equal(small, data[int(f):int(f) + 4096]), f"{kind}: random {name} read differs"
        rows.append(dict(base, measure="random_4KiB", method=name, reads=count, total_ms=round(ms, 1), per_read_ms=round(ms / count, 3),
                         per_1000_reads_ms=round(ms / count * 1000, 1)))
    h_enc = enc[:m].cpu().numpy()
    h_idx = idx[:ilen].cpu().numpy()
    h_out = np.empty(MIB, np.uint8)
    written = ctypes.c_uint64(0)
    for where, first in (("start", 0), ("end", n - MIB)):
        call = lambda: lib.density_b200_chameleon_decode_range_indexed(h_enc.ctypes.data, m, h_idx.ctypes.data, ilen, first,   # noqa: E731
                                                                       h_out.ctypes.data, MIB, ctypes.byref(written))
        for _ in range(2):
            assert call() == 0
        t0 = time.perf_counter()
        for _ in range(reps):
            call()
        ms = (time.perf_counter() - t0) * 1e3 / reps
        assert written.value == MIB and (h_out == data[first:first + MIB].cpu().numpy()).all()
        rows.append(dict(base, measure="sync_pageable_1MiB", interval=16 * MIB, window=where, indexed_ms=round(ms, 3)))
    del data, enc, idx
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--random-plain", type=int, default=100)
    args = ap.parse_args()
    lib = density_b200.load()
    print(json.dumps(card()), flush=True)
    for kind, n in (("text", GIB), ("mixed", 256 * MIB), ("noise", 256 * MIB)):
        for row in workload(lib, kind, n, args.reps, args.random_plain):
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
