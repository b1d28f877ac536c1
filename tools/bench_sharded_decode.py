"""Sharded Chameleon decode throughput: each rank decodes its piece of one sharded stream (density_b200_decode_sharded).

    torchrun --nproc_per_node N tools/bench_sharded_decode.py      (N GPUs, NCCL)
    python tools/bench_sharded_decode.py                           (one GPU)

Each rank takes 1 GiB of synth_text (first_page offset by rank, as the 2-rank test does), encodes it with encode_sharded without
a gather, then times decode_sharded between CUDA events (3 warm-ups, 20 steps). Rates are in uncompressed bytes. The decoded
shard is compared with the input on every rank outside the timed region. Rank 0 also times decode_device on its own piece, the
one-device comparison. One JSON line from rank 0.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_name_and_power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[torch.cuda.current_device()].split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=1 << 30, help="uncompressed bytes per rank")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench_sharded_decode needs a CUDA device")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import density_b200
    from density_b200 import sharded, synth
    lib = density_b200.load()
    n = args.bytes
    enc = sharded.ShardedEncoder(dev)
    dec = sharded.ShardedDecoder(dev)
    d_in = synth.synth_text(n, device=dev, first_page=rank * (n // synth.PAGE))
    d_enc = torch.empty(density_b200.Chameleon.safe_encode_buffer_size(n), dtype=torch.uint8, device=dev)
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    enc.encode(d_in, d_enc, d_sz, d_fl)
    torch.cuda.synchronize()
    if int(d_fl.item()):
        raise SystemExit("the sharded encode refused the stream")
    piece = d_enc[:int(d_sz.item())]
    d_dec = torch.empty(n, dtype=torch.uint8, device=dev)
    ms = timed(lambda: dec.decode(piece, d_dec, d_sz, d_fl), args.steps, args.warmup)
    ok = int(d_fl.item()) == 0 and int(d_sz.item()) == n and int(dec.d_total.item()) == world * n and torch.equal(d_dec, d_in)
    slowest = torch.tensor([ms], dtype=torch.float64, device=dev)
    okt = torch.tensor([0 if ok else 1], dtype=torch.int32, device=dev)
    if world > 1:
        dist.all_reduce(slowest, op=dist.ReduceOp.MAX)
        dist.all_reduce(okt, op=dist.ReduceOp.MAX)
    result = None
    if rank == 0:
        d_ref = torch.empty(n, dtype=torch.uint8, device=dev)
        ref_sz = torch.zeros(1, dtype=torch.int64, device=dev)
        stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        one = lambda: lib.density_b200_decode_device(0, piece.data_ptr(), piece.numel(), d_ref.data_ptr(), n, ref_sz.data_ptr(), stream())
        ms_one = timed(one, args.steps, args.warmup)
        ok_one = int(ref_sz.item()) == n and torch.equal(d_ref, d_in)
        name, power = gpu_name_and_power_limit()
        result = {
            "metric": "sharded_chameleon_decode",
            "gpus": world,
            "bytes_per_rank": n,
            "compressed_bytes_rank0": piece.numel(),
            "rank0_ms": round(ms, 4),
            "per_rank_GBps": round(n / ms / 1e6, 2),
            "aggregate_GBps": round(world * n / float(slowest.item()) / 1e6, 2),
            "decode_device_ms": round(ms_one, 4),
            "decode_device_GBps": round(n / ms_one / 1e6, 2),
            "correct": bool(okt.item() == 0) and ok_one,
            "gpu": name,
            "power_limit": power,
            "steps": args.steps,
            "warmup": args.warmup,
        }
        print(json.dumps(result), flush=True)
    if world > 1:
        dist.barrier()
    dec.close()
    enc.close()
    if world > 1:
        dist.destroy_process_group()
    if result is not None and not result["correct"]:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
