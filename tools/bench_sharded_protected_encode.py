"""Sharded Chameleon encode with copy mode: each rank encodes its shard of one stream (density_b200_encode_sharded_protected).

    torchrun --nproc_per_node N tools/bench_sharded_protected_encode.py      (N GPUs, NCCL)
    python tools/bench_sharded_protected_encode.py                           (one GPU)

Three inputs per rank, timed between CUDA events (warm-ups, then --steps steps) without a gather:
  mixed  --mixed-bytes of synth_mixed (text with embedded compressed and random regions: copy mode in many places)
  noise  --mixed-bytes of random bytes (copy mode everywhere)
  text   --text-bytes of synth_text (quiet: the round-0 verdict settles the map, so this is the cost of the path over the quiet one)
Rank 0 compares mixed and noise with encode_device (path 0, the single-device encoder: the whole copy-map iteration on one GPU) and text
with density_b200_encode_sharded (the quiet-only path; a collective, so every rank times it and the slowest rank's times are
compared). At N = 1 every piece is compared with encode_device's output outside the timed
region. It also reports the rounds the iteration used on rank 0 (ShardedChameleonEncoder.encode_protected, the phase API, run once).
Rates are in uncompressed bytes. One JSON line per input from rank 0.
"""
import argparse
import ctypes
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_sharded_cl_encode import gpu_name_and_power_limit, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mixed-bytes", type=int, default=256 << 20, help="bytes per rank of the mixed and noise inputs")
    ap.add_argument("--text-bytes", type=int, default=1 << 30, help="bytes per rank of the text input")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench_sharded_protected_encode needs a CUDA device")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import density_b200
    from density_b200 import sharded, synth
    lib = density_b200.load()
    enc = sharded.ShardedEncoder(dev)
    name, power = gpu_name_and_power_limit() if rank == 0 else (None, None)
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    bad = False
    inputs = (("mixed", lambda n: synth.synth_mixed(n, device=dev, first_region=rank * 64), args.mixed_bytes),
              ("noise", lambda n: synth.random_bytes(n, 1234 + rank, device=dev), args.mixed_bytes),
              ("text", lambda n: synth.synth_text(n, device=dev, first_page=rank * (n // synth.PAGE)), args.text_bytes))
    for label, make, n in inputs:
        d_in = make(n)
        cap = lib.chameleon_safe_encode_buffer_size(n)
        d_out = torch.empty(cap, dtype=torch.uint8, device=dev)
        d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
        d_fl = torch.ones(1, dtype=torch.int32, device=dev)
        ms = timed(lambda: enc.encode_protected(d_in, d_out, d_sz, d_fl), args.steps, args.warmup)
        flags = int(d_fl.item())
        stages = enc.profile()
        slowest = torch.tensor([ms], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(slowest, op=dist.ReduceOp.MAX)
        pe = sharded.ShardedChameleonEncoder()
        d_out2 = torch.empty(cap, dtype=torch.uint8, device=dev)
        d_sz2 = torch.zeros(1, dtype=torch.int64, device=dev)
        flags2, _, _ = pe.encode_protected(d_in, d_out2, d_sz2)
        status = pe.prot_status()
        pe.close()
        d_ref = torch.empty(cap, dtype=torch.uint8, device=dev)
        ref_sz = torch.zeros(1, dtype=torch.int64, device=dev)
        if label == "text":         # the quiet-only sharded path on the same shards: a collective, so every rank runs it
            ref_fl = torch.ones(1, dtype=torch.int32, device=dev)
            ms_base = timed(lambda: enc.encode(d_in, d_ref, ref_sz, ref_fl), args.steps, args.warmup)
            base_slowest = torch.tensor([ms_base], dtype=torch.float64, device=dev)
            if world > 1:
                dist.all_reduce(base_slowest, op=dist.ReduceOp.MAX)
            ms_base = float(base_slowest.item())
            ms_cmp = float(slowest.item())
            base_name = "encode_sharded"
            bad |= int(ref_fl.item()) != 0
        elif rank == 0:             # the single-device encoder with its copy-map iteration, on rank 0 only (no collective)
            base = lambda: lib.density_b200_encode_device_path(0, d_in.data_ptr(), n, d_ref.data_ptr(), cap, ref_sz.data_ptr(), stream(), 0)
            ms_base = timed(base, args.steps, args.warmup)
            ms_cmp = ms
            base_name = "encode_device"
        if rank == 0:
            m = int(ref_sz.item())
            correct = flags == 0 and flags2 == 0 and m > 0
            if world == 1:
                one_sz = torch.zeros(1, dtype=torch.int64, device=dev)
                one = torch.empty(cap, dtype=torch.uint8, device=dev)
                density_b200.encode_device("chameleon", d_in, one, one_sz)
                k = int(one_sz.item())
                correct = correct and int(d_sz.item()) == k and torch.equal(d_out[:k], one[:k]) and int(d_sz2.item()) == k \
                    and torch.equal(d_out2[:k], one[:k]) and m == k
            bad |= not correct
            print(json.dumps({
                "metric": f"sharded_protected_encode_{label}",
                "gpus": world,
                "bytes_per_rank": n,
                "compressed_bytes_rank0": int(d_sz.item()),
                "encode_sharded_protected_ms": round(ms, 4),
                "per_rank_GBps": round(n / ms / 1e6, 2),
                "aggregate_GBps": round(world * n / float(slowest.item()) / 1e6, 2),
                f"{base_name}_ms": round(ms_base, 4),
                f"{base_name}_GBps": round(n / ms_base / 1e6, 2),
                f"overhead_vs_{base_name}": round(ms_cmp / ms_base - 1.0, 4),
                "rounds_used": status["rounds"],
                "stage_ms": {k: round(v, 4) for k, v in zip(("phase1", "exchange_fold", "rounds_sizes_scan", "emit", "seams_gather"), stages)},
                "verdict": flags,
                "correct": correct,
                "gpu": name,
                "power_limit": power,
                "steps": args.steps,
                "warmup": args.warmup,
            }), flush=True)
        del d_in, d_out, d_out2
        torch.cuda.empty_cache()
    if world > 1:
        dist.barrier()
    enc.close()
    if world > 1:
        dist.destroy_process_group()
    if bad:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
