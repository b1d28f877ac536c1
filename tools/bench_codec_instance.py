"""Time CodecInstance encode / decode with pageable numpy buffers, host clock around each synchronous call.

Rows: Chameleon encode of 256 MiB of synth_text (the run-parallel kernels, so the host <-> device copies are a visible share of the
call), and Chameleon decode, Cheetah and Lion encode and decode of 16 MiB (the in-order kernel on the instance's state, where the
copies are a small share). Each call starts from a cleared instance, so every call does the same work. Prints the card's name and power
limit, then one JSON line per row: the mean and the best of --reps calls after one warm-up, in ms and GB/s of uncompressed bytes.
Usage: python tools/bench_codec_instance.py [--reps R]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from density_b200 import CODECS, synth  # noqa: E402
from density_b200.codec import CodecInstance  # noqa: E402

MIB = 1 << 20
ROWS = [("chameleon", "encode", 256 * MIB), ("chameleon", "decode", 16 * MIB), ("cheetah", "encode", 16 * MIB),
        ("cheetah", "decode", 16 * MIB), ("lion", "encode", 16 * MIB), ("lion", "decode", 16 * MIB)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_codec_instance.py needs a CUDA device")
    print(json.dumps(card()), flush=True)
    for alg, op, n in ROWS:
        text = synth.synth_text(n).numpy()
        C = CODECS[alg]
        enc = np.empty(C.safe_encode_buffer_size(n), np.uint8)
        enc = enc[:C.encode(text, enc)].copy()
        src, out = (text, np.empty(enc.size + n, np.uint8)) if op == "encode" else (enc, np.empty(n, np.uint8))
        want = enc if op == "encode" else text
        inst = CodecInstance(alg)
        ms = []
        for k in range(args.reps + 1):
            inst.clear_state()
            t0 = time.perf_counter()
            r = getattr(inst, op)(src, out)
            t = (time.perf_counter() - t0) * 1e3
            assert r == want.size and (out[:r] == want).all(), f"{alg} {op}: differs from the stateless call"
            if k:
                ms.append(t)
        mean = sum(ms) / len(ms)
        print(json.dumps({"alg": alg, "op": op, "bytes": n, "ms_mean": round(mean, 3), "ms_best": round(min(ms), 3),
                          "gbps_mean": round(n / mean / 1e6, 3), "gbps_best": round(n / min(ms) / 1e6, 3)}), flush=True)
        inst.close()


if __name__ == "__main__":
    main()
