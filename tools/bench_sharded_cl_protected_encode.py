"""Sharded Cheetah / Lion encode with copy mode on every shard (density_b200_encode_sharded_cl_protected), on one GPU.

    python tools/bench_sharded_cl_protected_encode.py [--shards 4] [--steps 3] [--warmup 1]

Per algorithm, three inputs, timed between CUDA events (warm-ups, then --steps steps) without a gather:
  text   --text-bytes of synth_text (quiet apart from the cold-dictionary start)
  mixed  --mixed-bytes of synth_mixed (text with embedded compressed and random regions: copy mode in many places)
  noise  --mixed-bytes of random bytes (copy mode everywhere)
Each runs through the NCCL driver at N = 1 and through the phase API (density_b200_cl_shard_prot_*) with --shards shards on the same
GPU, the exchanges done by stacking and the device folds. Baselines: encode_device on path 1 (the run-parallel encoder), or path 0
where path 1 does not settle its copy map; on text also density_b200_encode_sharded_cl, the quiet-only path, at N = 1. Every output is
compared with encode_device's outside the timed region. Reports the rounds until the map settled, ms and GB/s (uncompressed bytes), the
GPU name and its power limit. One JSON line per algorithm and input.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_sharded_cl_encode import gpu_name_and_power_limit, timed  # noqa: E402


class PhaseShards:
    """W shards of one input on one GPU through the phase API; run() enqueues one whole encode on torch's current stream."""

    def __init__(self, lib, alg, d_in, world):
        from density_b200 import sharded as S
        self.S, self.lib, self.alg, self.world = S, lib, alg, world
        n = d_in.numel()
        cuts = [n * r // world // 256 * 256 for r in range(world)] + [n]
        self.cuts = cuts
        self.ins = [d_in[cuts[r]:cuts[r + 1]] for r in range(world)]
        self.encs = [S.ShardedCLEncoder(alg) for _ in range(world)]
        dev = d_in.device
        wp, wc = self.encs[0].words_p, self.encs[0].words_c
        self.words = torch.zeros((world, S.CL_PROT_ROUND_WORDS), dtype=torch.int32, device=dev)
        self.tp = torch.zeros((world, wp), dtype=torch.int32, device=dev)
        self.tc = torch.zeros((world, wc), dtype=torch.int32, device=dev)
        self.tr = torch.zeros((world, S.PROT_TRANSFER_WORDS), dtype=torch.int32, device=dev)
        self.seams = torch.zeros((world, S.SEAM_WORDS), dtype=torch.int32, device=dev)
        safe = getattr(lib, f"{alg}_safe_encode_buffer_size")
        self.caps = [safe(x.numel()) for x in self.ins]
        self.outs = [torch.empty(c, dtype=torch.uint8, device=dev) for c in self.caps]
        self.sizes = torch.zeros((world,), dtype=torch.int64, device=dev)

    def run(self):
        S, lib, W, e = self.S, self.lib, self.world, self.encs
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        a = S._alg_id(self.alg)

        def ok(rc):
            assert rc == 0, lib.density_b200_last_error()
        for r in range(W):
            ok(lib.density_b200_cl_shard_prot_phase1(e[r]._h, self.ins[r].data_ptr(), self.ins[r].numel(), self.cuts[r], int(r == W - 1),
                                                     self.words[r].data_ptr(), st))
        for _ in range(lib.density_b200_prot_round_budget()):
            for r in range(W):
                ok(lib.density_b200_cl_shard_prot_p(e[r]._h, self.words.data_ptr(), W, r, self.tp[r].data_ptr(), st))
            cp = [S.fold_cl_tables(a, S.CL_TABLE_P, self.tp, r) for r in range(W)]
            for r in range(W):
                ok(lib.density_b200_cl_shard_prot_c(e[r]._h, cp[r].data_ptr(), self.tc[r].data_ptr(), st))
            cc = [S.fold_cl_tables(a, S.CL_TABLE_C, self.tc, r) for r in range(W)]
            for r in range(W):
                ok(lib.density_b200_cl_shard_prot_transfer(e[r]._h, cc[r].data_ptr(), self.tr[r].data_ptr(), st))
            for r in range(W):
                ok(lib.density_b200_cl_shard_prot_settle(e[r]._h, self.tr.data_ptr(), W, r, self.words[r].data_ptr(), st))
            for r in range(W):
                ok(lib.density_b200_cl_shard_prot_next(e[r]._h, self.words.data_ptr(), W, st))
        for r in range(W):
            ok(lib.density_b200_cl_shard_prot_finish(e[r]._h, self.outs[r].data_ptr(), self.caps[r], self.sizes[r:].data_ptr(),
                                                     self.seams[r].data_ptr(), st))

    def result(self):
        """(verdict, concatenated pieces, rounds)"""
        flags, _, _ = self.S.seam_verdict(self.seams)
        sz = self.sizes.tolist()
        cat = torch.cat([self.outs[r][:sz[r]] for r in range(self.world)])
        return flags, cat, self.encs[0].prot_status()["rounds"]

    def close(self):
        for x in self.encs:
            x.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--text-bytes", type=int, default=1 << 30)
    ap.add_argument("--mixed-bytes", type=int, default=256 << 20, help="bytes of the mixed and noise inputs")
    ap.add_argument("--shards", type=int, default=4, help="shards on one GPU through the phase API")
    ap.add_argument("--algs", default="cheetah,lion")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sharded_cl_protected_encode needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import density_b200
    from density_b200 import sharded, synth
    lib = density_b200.load()
    name, power = gpu_name_and_power_limit()
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    enc = sharded.ShardedEncoder(dev)
    bad = False
    inputs = (("text", lambda n: synth.synth_text(n, device=dev), args.text_bytes),
              ("mixed", lambda n: synth.synth_mixed(n, device=dev), args.mixed_bytes),
              ("noise", lambda n: synth.random_bytes(n, 1234, device=dev), args.mixed_bytes))
    for alg in args.algs.split(","):
        a = sharded._alg_id(alg)
        for label, make, n in inputs:
            d_in = make(n)
            cap = getattr(lib, f"{alg}_safe_encode_buffer_size")(n)
            # the single-device encoder: path 1, or path 0 (with its in-order fallback) when path 1 does not settle
            d_ref = torch.empty(cap, dtype=torch.uint8, device=dev)
            ref_sz = torch.zeros(1, dtype=torch.int64, device=dev)
            path = 1
            base = lambda: lib.density_b200_encode_device_path(a, d_in.data_ptr(), n, d_ref.data_ptr(), cap, ref_sz.data_ptr(), stream(), path)
            base()
            torch.cuda.synchronize()
            if int(ref_sz.item()) == 0:
                path = 0
            ms_dev = timed(base, args.steps, args.warmup)
            k = int(ref_sz.item())
            # the NCCL driver at N = 1
            d_out = torch.empty(cap, dtype=torch.uint8, device=dev)
            d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
            d_fl = torch.ones(1, dtype=torch.int32, device=dev)
            ms_one = timed(lambda: enc.encode_protected(d_in, d_out, d_sz, d_fl, alg=alg), args.steps, args.warmup)
            stages = enc.profile()
            one_ok = int(d_fl.item()) == 0 and int(d_sz.item()) == k and torch.equal(d_out[:k], d_ref[:k])
            del d_out
            # W shards through the phase API
            ps = PhaseShards(lib, alg, d_in, args.shards)
            ms_w = timed(ps.run, args.steps, args.warmup)
            flags, cat, rounds = ps.result()
            w_ok = flags == 0 and cat.numel() == k and torch.equal(cat, d_ref[:k])
            ps.close()
            del cat
            row = {
                "metric": f"sharded_cl_protected_encode_{alg}_{label}",
                "bytes": n,
                "compressed_bytes": k,
                "encode_device_path": path,
                "encode_device_ms": round(ms_dev, 4),
                "encode_device_GBps": round(n / ms_dev / 1e6, 2),
                "n1_ms": round(ms_one, 4),
                "n1_GBps": round(n / ms_one / 1e6, 2),
                "n1_stage_ms": {s: round(v, 4) for s, v in zip(("phase1", "exchange_fold", "rounds_sizes_scan", "emit", "seams_gather"), stages)},
                f"shards{args.shards}_one_gpu_ms": round(ms_w, 4),
                f"shards{args.shards}_one_gpu_GBps": round(n / ms_w / 1e6, 2),
                f"shards{args.shards}_rounds_used": rounds,
            }
            if label == "text":    # the quiet-only sharded path on the same input
                q_out = torch.empty(cap, dtype=torch.uint8, device=dev)
                q_sz = torch.zeros(1, dtype=torch.int64, device=dev)
                q_fl = torch.ones(1, dtype=torch.int32, device=dev)
                ms_q = timed(lambda: enc.encode(d_in, q_out, q_sz, q_fl, alg=alg), args.steps, args.warmup)
                row["encode_sharded_cl_ms"] = round(ms_q, 4)
                row["n1_overhead_vs_encode_sharded_cl"] = round(ms_one / ms_q - 1.0, 4)
                one_ok = one_ok and int(q_fl.item()) == 0
                del q_out
            row.update({"correct": one_ok and w_ok, "gpu": name, "power_limit": power, "steps": args.steps, "warmup": args.warmup})
            bad |= not row["correct"]
            print(json.dumps(row), flush=True)
            del d_in, d_ref
            torch.cuda.empty_cache()
    enc.close()
    if bad:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
