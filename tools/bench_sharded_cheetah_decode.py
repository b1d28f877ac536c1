"""Sharded Cheetah decode throughput: each rank decodes its piece of one stream (density_b200_decode_sharded_cheetah).

    torchrun --nproc_per_node N tools/bench_sharded_cheetah_decode.py      (N GPUs, NCCL)
    python tools/bench_sharded_cheetah_decode.py                           (one GPU)

Each rank takes --bytes of synth_text (first_page offset by rank), encodes it with ShardedEncoder(alg="cheetah") and times
ShardedDecoder.decode(alg="cheetah") on its piece between CUDA events (--warmup warm-ups, then --steps steps). Rank 0 also times:
  - decode_device on its own piece, the one-device comparison (at N = 1 the same stream), and its round count;
  - the phase API with --pieces pieces of that stream on one GPU (the slices at the stream offsets of equal shard cuts), the exchanges
    replaced by the library's folds: total time per step, the rounds until settled, and per round the time of the walks with their
    exports and of the folds (CUDA events); the rounds after the settled one are gated off on the device, and their time is the cost
    of the gated rounds;
  - one phase-API step under torch.profiler: the summed time of every kernel, by name (cd_pred_export is the per-round export).
Every decoded piece is compared with the input outside the timed region. Rates are in uncompressed bytes. One JSON line from rank 0.
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


class Pieces:
    """The phase API over the pieces of one stream on one GPU (what tests/test_gpu_sharded_cheetah_decode.py drives)."""

    def __init__(self, lib, d_enc, cuts, caps, dev):
        from density_b200 import sharded
        self.lib, self.sharded, self.cuts, self.caps = lib, sharded, cuts, caps
        self.world = len(cuts) - 1
        self.ins = [d_enc[cuts[r]:cuts[r + 1]] for r in range(self.world)]
        self.outs = [torch.empty(caps[r], dtype=torch.uint8, device=dev) for r in range(self.world)]
        self.hs = [lib.density_b200_cheetah_decode_shard_create() for _ in range(self.world)]
        self.tc = torch.zeros((self.world, lib.density_b200_cheetah_cmap_words()), dtype=torch.int32, device=dev)
        self.tp = torch.zeros((self.world, lib.density_b200_cl_table_words(1, sharded.CL_TABLE_P)), dtype=torch.int32, device=dev)
        self.words = torch.zeros((self.world, 4), dtype=torch.int32, device=dev)
        self.seam = torch.zeros((self.world, 8), dtype=torch.int32, device=dev)
        self.sizes = torch.zeros(self.world, dtype=torch.int64, device=dev)
        self.budget = lib.density_b200_cheetah_decode_round_budget()
        self.ev = None

    def step(self, events=False):
        L, sh, W = self.lib, self.sharded, self.world
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3 + 2 * self.budget)] if events else None
        mark = (lambda k: ev[k].record()) if events else (lambda k: None)
        rc = 0
        mark(0)
        for r in range(W):
            rc |= L.density_b200_cheetah_decode_shard_phase1(self.hs[r], self.ins[r].data_ptr(), self.ins[r].numel(), self.outs[r].data_ptr(),
                                                             self.caps[r], int(r == 0), int(r == W - 1), self.tc[r].data_ptr(), st)
        for r in range(W):
            carry = sh.fold_cheetah_cmap(self.tc, r) if r > 0 else None
            rc |= L.density_b200_cheetah_decode_shard_phase2(self.hs[r], carry.data_ptr() if carry is not None else None, st)
        mark(1)
        for k in range(self.budget):
            for r in range(W):
                rc |= L.density_b200_cheetah_decode_shard_round_walk(self.hs[r], self.tp[r].data_ptr(), self.words[r].data_ptr(), st)
            mark(2 + 2 * k)
            for r in range(W):
                carry = sh.fold_cl_tables("cheetah", sh.CL_TABLE_P, self.tp, r) if r > 0 else None
                rc |= L.density_b200_cheetah_decode_shard_round_fold(self.hs[r], carry.data_ptr() if carry is not None else None,
                                                                     self.words.data_ptr(), W, r, st)
            mark(3 + 2 * k)
        for r in range(W):
            rc |= L.density_b200_cheetah_decode_shard_phase3(self.hs[r], self.sizes[r:r + 1].data_ptr(), self.seam[r].data_ptr(), st)
        mark(2 + 2 * self.budget)
        if rc:
            raise RuntimeError(f"phase API rc={rc}: {L.density_b200_last_error().decode()}")
        self.ev = ev

    def rounds(self):
        s4 = (ctypes.c_uint32 * 4)()
        assert self.lib.density_b200_cheetah_decode_shard_status(self.hs[0], s4) == 0
        return int(s4[0]), int(s4[1])

    def close(self):
        for h in self.hs:
            self.lib.density_b200_cheetah_decode_shard_destroy(h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=1 << 30, help="uncompressed bytes per rank")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pieces", type=int, default=4, help="pieces of the phase-API run on one GPU")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench_sharded_cheetah_decode needs a CUDA device")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import density_b200
    from density_b200 import sharded, synth
    lib = density_b200.load()
    n = args.bytes
    d_in = synth.synth_text(n, device=dev, first_page=rank * (n // synth.PAGE))
    cap_enc = lib.cheetah_safe_encode_buffer_size(n)
    d_enc = torch.empty(cap_enc, dtype=torch.uint8, device=dev)
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    enc = sharded.ShardedEncoder(dev)
    enc.encode(d_in, d_enc, d_sz, d_fl, alg="cheetah")
    torch.cuda.synchronize()
    m = int(d_sz.item())
    assert int(d_fl.item()) == 0, "the sharded encode refused the input"
    piece = d_enc[:m].clone()
    del d_enc
    dec = sharded.ShardedDecoder(dev)
    d_out = torch.empty(n + 64, dtype=torch.uint8, device=dev)
    d_osz = torch.zeros(1, dtype=torch.int64, device=dev)
    ms = timed(lambda: dec.decode(piece, d_out, d_osz, d_fl, alg="cheetah"), args.steps, args.warmup)
    flags = int(d_fl.item())
    correct = flags == 0 and int(d_osz.item()) == n and torch.equal(d_out[:n], d_in)
    slowest = torch.tensor([ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(slowest, op=dist.ReduceOp.MAX)
    if rank == 0:
        name, power = gpu_name_and_power_limit()
        # decode_device on the same piece: at N = 1 the whole stream
        one = lambda: density_b200.decode_device("cheetah", piece, m, d_out, d_osz)
        ms_one = timed(one, args.steps, args.warmup)
        ok_one = int(d_osz.item()) == n and torch.equal(d_out[:n], d_in)
        r4 = (ctypes.c_uint32 * 4)()
        rounds_one = int(r4[0]) if lib.density_b200_cheetah_decode_rounds(r4) == 0 else None
        res = {
            "metric": "sharded_cheetah_decode",
            "gpus": world,
            "bytes_per_rank": n,
            "compressed_bytes_rank0": m,
            "decode_sharded_cheetah_ms": round(ms, 3),
            "per_rank_GBps": round(n / ms / 1e6, 3),
            "aggregate_GBps": round(world * n / float(slowest.item()) / 1e6, 3),
            "decode_device_ms": round(ms_one, 3),
            "decode_device_GBps": round(n / ms_one / 1e6, 3),
            "decode_device_rounds": rounds_one,
            "overhead_vs_decode_device": round(ms / ms_one - 1.0, 4) if world == 1 else None,
        }
        del d_out
        # the phase API with --pieces pieces of one stream on this GPU (rank 0's stream at N = 1)
        W = args.pieces
        per = n // W // 256 * 256
        shard_cuts = [r * per for r in range(W)] + [n]
        stream_cuts = [0]
        for c in shard_cuts[1:-1]:         # a prefix of a multiple of 256 bytes encodes to a prefix of the stream
            tmp = torch.empty(lib.cheetah_safe_encode_buffer_size(c), dtype=torch.uint8, device=dev)
            density_b200.encode_device("cheetah", d_in[:c], tmp, d_sz)
            torch.cuda.synchronize()
            stream_cuts.append(int(d_sz.item()))
            del tmp
        stream_cuts.append(m)
        P = Pieces(lib, piece, stream_cuts, [shard_cuts[r + 1] - shard_cuts[r] + 64 for r in range(W)], dev)
        ms_ph = timed(P.step, args.steps, args.warmup)
        P.step(events=True)
        torch.cuda.synchronize()
        used, settled = P.rounds()
        ev = P.ev
        walk = [ev[1 + 2 * k].elapsed_time(ev[2 + 2 * k]) for k in range(P.budget)]
        fold = [ev[2 + 2 * k].elapsed_time(ev[3 + 2 * k]) for k in range(P.budget)]
        ok_ph = settled == 1 and int(P.seam[:, 2].sum().item()) == 0 and all(
            int(P.sizes[r].item()) == shard_cuts[r + 1] - shard_cuts[r] and torch.equal(P.outs[r][:shard_cuts[r + 1] - shard_cuts[r]],
                                                                                         d_in[shard_cuts[r]:shard_cuts[r + 1]]) for r in range(W))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            P.step()
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" and e.count:
                k = e.key.split("(")[0].split("<")[0].replace("void ", "").replace("dns::", "")
                kernels[k] = round(kernels.get(k, 0.0) + e.device_time_total / 1000.0, 3)
        P.close()
        res.update({
            "phase_pieces": W,
            "phase_total_ms": round(ms_ph, 3),
            "phase_GBps": round(n / ms_ph / 1e6, 3),
            "phase_rounds_until_settled": used,
            "phase_settled": settled,
            "phase_front_ms": round(ev[0].elapsed_time(ev[1]), 3),
            "phase_round_walk_export_ms": [round(x, 3) for x in walk],
            "phase_round_fold_ms": [round(x, 3) for x in fold],
            "phase_gated_rounds_ms": round(ev[2 * used + 1].elapsed_time(ev[2 * P.budget + 1]), 3),
            "phase_tail_ms": round(ev[2 * P.budget + 1].elapsed_time(ev[2 * P.budget + 2]), 3),
            "kernel_ms_one_step": dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:16]),
            "verdict": flags,
            "correct": bool(correct and ok_one and ok_ph),
            "gpu": name,
            "power_limit": power,
            "steps": args.steps,
            "warmup": args.warmup,
        })
        print(json.dumps(res), flush=True)
        correct = res["correct"]
    if world > 1:
        dist.barrier()
    enc.close(); dec.close()
    if world > 1:
        dist.destroy_process_group()
    if not correct:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
