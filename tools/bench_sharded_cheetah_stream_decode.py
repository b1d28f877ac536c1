"""Sharded Cheetah decode of a stream without known cuts (density_b200_decode_sharded_cheetah_stream): each rank finds its piece.

    torchrun --nproc_per_node N tools/bench_sharded_cheetah_stream_decode.py      (N GPUs, NCCL)
    python tools/bench_sharded_cheetah_stream_decode.py                           (one GPU)

Every rank makes the same N x 1 GiB of synth_text and encodes it with ONE cheetah_encode call (density_b200_encode_device), then
keeps its range + halo of that stream (sharded.stream_ranges). Timed between CUDA events (3 warm-ups, 20 steps):
  locate_start_ms      the range map of rank 0's range as the range that holds the stream start: the exact boundary walk over range
                       + halo (9 kernels) and the start row
  locate_candidate_ms  the range map of the same range as a later range: candidate walks, group and range composition
  piece_ms             density_b200_decode_sharded_cheetah on the located piece, the cuts known beforehand
  stream_ms            density_b200_decode_sharded_cheetah_stream: locate, map all-gather, host round trip, then the piece decode
  decode_device_ms     (N = 1) density_b200_decode_device on the same stream
stream_ms - piece_ms is what finding the cuts costs. Rates are in uncompressed bytes; the decoded pieces are checked against the
input at their offsets outside the timed region. One JSON line from rank 0.
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

from tools.bench_sharded_decode import gpu_name_and_power_limit, timed  # noqa: E402


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
        raise SystemExit("bench_sharded_cheetah_stream_decode needs a CUDA device")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import density_b200
    from density_b200 import sharded, synth
    lib = density_b200.load()
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    total = world * args.bytes
    d_data = synth.synth_text(total, device=dev)
    d_enc = torch.empty(density_b200.Cheetah.safe_encode_buffer_size(total), dtype=torch.uint8, device=dev)
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    if lib.density_b200_encode_device(1, d_data.data_ptr(), total, d_enc.data_ptr(), d_enc.numel(), d_sz.data_ptr(), stream()):
        raise SystemExit(f"encode failed: {lib.density_b200_last_error().decode()}")
    torch.cuda.synchronize()
    m = int(d_sz.item())
    o, n_range, n_halo = sharded.stream_ranges(m, world)[rank]
    d_in = d_enc[o:o + n_range + n_halo].clone()
    cap = min(16 * (n_range + n_halo), total + 64)      # 16x always fits a quiet piece; no piece decodes to more than the input
    d_out = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    dec = sharded.ShardedDecoder(dev)
    loc = lib.density_b200_cheetah_decode_shard_create()
    d_map = torch.empty(sharded.CHEETAH_LOCATE_MAP_WORDS, dtype=torch.int64, device=dev)
    locate = lambda off: lib.density_b200_cheetah_decode_locate(loc, d_in.data_ptr(), n_range, n_halo, off, d_map.data_ptr(), stream())
    locate_start_ms = timed(lambda: locate(0), args.steps, args.warmup)
    locate_candidate_ms = timed(lambda: locate(o if o else n_range), args.steps, args.warmup)
    locate(o)                                                   # this rank's own map, for the known-cut piece below
    stream_ms = timed(lambda: dec.decode_stream(d_in, n_range, d_out, d_sz, d_fl, alg="cheetah", range_offset=o), args.steps, args.warmup)
    off, k = int(dec.d_offset.item()), int(d_sz.item())
    ok = int(d_fl.item()) == 0 and int(dec.d_total.item()) == total and torch.equal(d_out[:k], d_data[off:off + k])
    # the same piece with its cuts known beforehand
    if world > 1:
        maps = torch.empty((world, sharded.CHEETAH_LOCATE_MAP_WORDS), dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(maps.view(-1), d_map)
    else:
        maps = d_map.view(1, -1)
    start, end, _, _, _ = sharded.locate_piece(maps.cpu().numpy().view("uint64"), rank, alg="cheetah")
    piece = d_in[start:end].clone()
    piece_ms = timed(lambda: dec.decode(piece, d_out, d_sz, d_fl, alg="cheetah"), args.steps, args.warmup)
    ok = ok and int(d_fl.item()) == 0 and int(d_sz.item()) == k and torch.equal(d_out[:k], d_data[off:off + k])
    per = torch.tensor([locate_start_ms, locate_candidate_ms, piece_ms, stream_ms, k], dtype=torch.float64, device=dev)
    okt = torch.tensor([0 if ok else 1], dtype=torch.int32, device=dev)
    if world > 1:
        dist.all_reduce(per, op=dist.ReduceOp.MAX)
        dist.all_reduce(okt, op=dist.ReduceOp.MAX)
    result = None
    if rank == 0:
        res = {}
        if world == 1:
            d_ref = torch.empty(total + 64, dtype=torch.uint8, device=dev)
            ref_sz = torch.zeros(1, dtype=torch.int64, device=dev)
            one = lambda: lib.density_b200_decode_device(1, d_enc.data_ptr(), m, d_ref.data_ptr(), d_ref.numel(), ref_sz.data_ptr(), stream())
            ms_one = timed(one, args.steps, args.warmup)
            ok = ok and int(ref_sz.item()) == total and torch.equal(d_ref[:total], d_data)
            res = {"decode_device_ms": round(ms_one, 4), "decode_device_GBps": round(total / ms_one / 1e6, 2)}
        name, power = gpu_name_and_power_limit()
        slowest = per.tolist()
        result = {
            "metric": "sharded_cheetah_stream_decode",
            "gpus": world,
            "bytes_per_rank": args.bytes,
            "compressed_bytes": m,
            "rank0_range_bytes": n_range,
            "locate_start_ms": round(locate_start_ms, 4),
            "locate_candidate_ms": round(locate_candidate_ms, 4),
            "piece_ms": round(piece_ms, 4),
            "stream_ms": round(stream_ms, 4),
            "find_cuts_ms": round(stream_ms - piece_ms, 4),
            "find_cuts_share_of_piece": round((stream_ms - piece_ms) / piece_ms, 4),
            "per_rank_GBps": round(k / stream_ms / 1e6, 2),
            "aggregate_GBps": round(total / slowest[3] / 1e6, 2),
            "slowest_rank_ms": {"locate_start": round(slowest[0], 4), "locate_candidate": round(slowest[1], 4), "piece": round(slowest[2], 4),
                                "stream": round(slowest[3], 4)},
            **res,
            "correct": bool(okt.item() == 0) and ok,
            "gpu": name,
            "power_limit": power,
            "steps": args.steps,
            "warmup": args.warmup,
        }
        print(json.dumps(result), flush=True)
    if world > 1:
        dist.barrier()
    lib.density_b200_cheetah_decode_shard_destroy(loc)
    dec.close()
    if world > 1:
        dist.destroy_process_group()
    if result is not None and not result["correct"]:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
