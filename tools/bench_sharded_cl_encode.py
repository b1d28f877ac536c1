"""Sharded Cheetah / Lion encode throughput: each rank encodes its shard of one stream (density_b200_encode_sharded_cl).

    torchrun --nproc_per_node N tools/bench_sharded_cl_encode.py      (N GPUs, NCCL)
    python tools/bench_sharded_cl_encode.py                           (one GPU)

Each rank takes --bytes of synth_text (first_page offset by rank, as the 2-rank test does) and times encode_sharded_cl without a
gather between CUDA events (warm-ups, then --steps steps), for Cheetah and Lion. Rank 0 also times encode_device (path 1, the
run-parallel encoder without the in-order kernel behind it) on its own shard, the one-device comparison, and the phases of the
phase-level encoder (ShardedCLEncoder: phase 1, P exchange + fold, phase 2, C exchange + fold, phase 3 + seams; one timed call after
the warm-ups). At N = 1 every piece is compared with encode_device's output outside the timed region. Rates are in uncompressed bytes.
One JSON line per algorithm from rank 0.
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
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--algs", default="cheetah,lion")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench_sharded_cl_encode needs a CUDA device")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import density_b200
    from density_b200 import sharded, synth
    lib = density_b200.load()
    n = args.bytes
    enc = sharded.ShardedEncoder(dev)
    d_in = synth.synth_text(n, device=dev, first_page=rank * (n // synth.PAGE))
    name, power = gpu_name_and_power_limit() if rank == 0 else (None, None)
    bad = False
    for alg in args.algs.split(","):
        aid = sharded.ALGS[alg]
        cap = getattr(lib, f"{alg}_safe_encode_buffer_size")(n)
        d_out = torch.empty(cap, dtype=torch.uint8, device=dev)
        d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
        d_fl = torch.ones(1, dtype=torch.int32, device=dev)
        ms = timed(lambda: enc.encode(d_in, d_out, d_sz, d_fl, alg=alg), args.steps, args.warmup)
        flags = int(d_fl.item())
        slowest = torch.tensor([ms], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(slowest, op=dist.ReduceOp.MAX)
        pe = sharded.ShardedCLEncoder(alg)
        d_out2 = torch.empty(cap, dtype=torch.uint8, device=dev)
        d_sz2 = torch.zeros(1, dtype=torch.int64, device=dev)
        for _ in range(args.warmup):
            pe.encode(d_in, d_out2, d_sz2)
        pe.encode(d_in, d_out2, d_sz2, timing=True)
        phases = pe.phase_ms()
        pe.close()
        if rank == 0:
            d_ref = torch.empty(cap, dtype=torch.uint8, device=dev)
            ref_sz = torch.zeros(1, dtype=torch.int64, device=dev)
            stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            one = lambda: lib.density_b200_encode_device_path(aid, d_in.data_ptr(), n, d_ref.data_ptr(), cap, ref_sz.data_ptr(), stream(), 1)
            ms_one = timed(one, args.steps, args.warmup)
            m = int(ref_sz.item())
            correct = flags == 0 and m > 0
            if world == 1:
                correct = correct and int(d_sz.item()) == m and torch.equal(d_out[:m], d_ref[:m]) and int(d_sz2.item()) == m \
                    and torch.equal(d_out2[:m], d_ref[:m])
            bad |= not correct
            print(json.dumps({
                "metric": f"sharded_{alg}_encode",
                "gpus": world,
                "bytes_per_rank": n,
                "compressed_bytes_rank0": int(d_sz.item()),
                "encode_sharded_cl_ms": round(ms, 4),
                "per_rank_GBps": round(n / ms / 1e6, 2),
                "aggregate_GBps": round(world * n / float(slowest.item()) / 1e6, 2),
                "encode_device_ms": round(ms_one, 4),
                "encode_device_GBps": round(n / ms_one / 1e6, 2),
                "overhead_vs_encode_device": round(ms / ms_one - 1.0, 4),
                "phase_ms": {k: round(v, 4) for k, v in zip(("phase1", "exchange_fold_p", "phase2", "exchange_fold_c", "phase3_seams"), phases)},
                "verdict": flags,
                "correct": correct,
                "gpu": name,
                "power_limit": power,
                "steps": args.steps,
                "warmup": args.warmup,
            }), flush=True)
    if world > 1:
        dist.barrier()
    enc.close()
    if world > 1:
        dist.destroy_process_group()
    if bad:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
