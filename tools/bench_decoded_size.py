"""Time the decoded-size query (density_b200_decoded_size_device) next to decode_device on the same stream, with CUDA events.

Workloads: 1 GiB of synthetic text encoded by each algorithm (a quiet stream: the in-order walk jumps whole groups of chunks), and
256 MiB of synth_mixed and of noise (copy-mode blocks: the walk goes through the dirty chunks block by block). decode_device is timed on
the same stream for comparison, except Lion on the 1 GiB text (its decode walks the prediction lists in order, about 20 s a GiB).
Prints the card's name and power limit first, then one JSON line per workload. Usage: python tools/bench_decoded_size.py [--reps R]"""
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


def workload(alg, kind, n, reps, with_decode):
    data = {"text": lambda: synth.synth_text(n, device="cuda"), "mixed": lambda: synth.synth_mixed(n, device="cuda"),
            "noise": lambda: synth.random_bytes(n, 5, device="cuda")}[kind]()
    enc = torch.empty(density_b200.CODECS[alg].safe_encode_buffer_size(n), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    codec.encode_device(alg, data, enc, sz)
    torch.cuda.synchronize()
    m = int(sz.item())
    res = torch.zeros(2, dtype=torch.int64, device="cuda")
    q_ms = timed(lambda: codec.decoded_size_device(alg, enc, m, res), 3, reps)
    assert res.cpu().tolist() == [n, 0], f"{alg} {kind}: the query says {res.cpu().tolist()}, the input was {n} bytes"
    row = {"alg": alg, "corpus": kind, "input_bytes": n, "stream_bytes": m, "query_ms": round(q_ms, 4),
           "query_stream_gbps": round(m / q_ms / 1e6, 2)}
    if with_decode:
        out = torch.empty(n, dtype=torch.uint8, device="cuda")
        d_ms = timed(lambda: codec.decode_device(alg, enc, m, out, sz), 1, max(1, reps // 5) if alg == "lion" else reps)
        assert int(sz.item()) == n and torch.equal(out, data), f"{alg} {kind}: decode differs"
        row.update(decode_ms=round(d_ms, 3), query_share_of_decode=round(q_ms / d_ms, 5))
        del out
    else:
        row.update(decode_ms=None)
    del data, enc
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    density_b200.load()
    print(json.dumps(card()), flush=True)
    for alg in ("chameleon", "cheetah", "lion"):
        print(json.dumps(workload(alg, "text", GIB, args.reps, alg != "lion")), flush=True)
        for kind in ("mixed", "noise"):
            print(json.dumps(workload(alg, kind, 256 * MIB, args.reps, True)), flush=True)


if __name__ == "__main__":
    main()
