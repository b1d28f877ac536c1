"""Static pipe counts of the full-tile path of the Chameleon flag pass `cham_flag_pass6` (DESIGN.md section 3), per phase.

Compiles `density_b200/csrc/chameleon_encode.cu` with the flags of `density_b200/build.py` (or takes `--sass` / `--src`), cuts the
SASS of `cham_flag_pass6` at its `BAR.SYNC`s and counts the warp instructions of every phase of a whole tile without copy-mode blocks
by pipe:
  FMA     IMAD* (the integer multiply-add unit, which issues beside the ALU pipe)
  MIO     LDS / STS / ATOMS / SHFL / VOTE / POPC / FLO / S2R / WARPSYNC / BAR (shared memory, warp-wide and special-register ops)
  branch  BRA / BSSY / BSYNC / EXIT / CALL / RET
  mem     LDG / STG / LDC
  ALU     everything else (ISETP, LOP3, SHF, SEL, IADD3, LEA, PRMT, VIMNMX, MOV, ...)
The per-tile layout the cut relies on (checked): the function has one barrier before the tile loop, four in the tile body for tiles
with copy-mode blocks or a partial tile, four in the whole-tile body, and one in `f6_replay`; the whole-tile body starts after the
first body's last barrier and the branch that leaves it, and the loop's back edge jumps to the per-tile prologue shared by the two.

Weights: the deposit loop (between S2 and S3) and the D loop (between S3 and S4) run ceil(records of the warp / 32) times, so their
bodies count that many times on average over the records per warp of the bench text, which `tools/proto_tile_protocol_v6.py` counts
(default: run 0 of the 1 GiB text, 496 tiles; `--trips` overrides). Loops nested in the D loop (the overflow mailboxes) are cold on
text and count 0 times; every other instruction counts once, the rare fingerprint-0 path of A included.

    python -m tools.sass_pipes [--src chameleon_encode.cu] [--sass file] [--trips 1.09]
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "_ZN3dns4cham15cham_flag_pass6"
PIPES = ("ALU", "FMA", "MIO", "branch", "mem")
MIO = ("LDS", "STS", "ATOMS", "SHFL", "VOTE", "VOTEU", "POPC", "FLO", "S2R", "S2UR", "WARPSYNC", "BAR", "MATCH", "REDUX")
BRANCH = ("BRA", "BSSY", "BSYNC", "EXIT", "CALL", "RET", "BREAK", "NOP")
MEM = ("LDG", "STG", "LDC", "ULDC")
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?);")


def pipe(op):
    base = op.split(".")[0]
    if base.startswith("IMAD"):
        return "FMA"
    if base in MIO:
        return "MIO"
    if base in BRANCH:
        return "branch"
    if base in MEM:
        return "mem"
    return "ALU"


def sass_of(src):
    sys.path.insert(0, ROOT)
    from density_b200 import build as b
    with tempfile.TemporaryDirectory() as d:
        obj = os.path.join(d, "ce.o")
        subprocess.run([b.nvcc_path()] + b.NVCC_FLAGS + ["-c", src, "-o", obj], check=True)
        return subprocess.run([os.path.join(os.path.dirname(b.nvcc_path()), "cuobjdump"), "-sass", obj], check=True,
                              capture_output=True, text=True).stdout


def parse(sass):
    out, on = [], False
    for line in sass.splitlines():
        if "Function : " in line:
            on = KERNEL in line
            continue
        m = INSN.search(line) if on else None
        if m:
            text = m.group(2).strip()
            pred = text.startswith("@")
            body = text.split(None, 1)[1] if pred else text
            op = body.split()[0]
            tgt = None
            if op.startswith("BRA") or op.startswith("BSSY"):
                t = re.findall(r"0x([0-9a-f]+)\s*$", body)
                tgt = int(t[0], 16) if t else None
            out.append((int(m.group(1), 16), op, tgt, text))
    return out


def cut(ins):
    bars = [k for k, x in enumerate(ins) if x[1].startswith("BAR.SYNC")]
    assert len(bars) == 10, f"expected 10 barriers in {KERNEL}, found {len(bars)}"
    addr = [x[0] for x in ins]
    # whole-tile body: after the first body's S4 and the unconditional branch that leaves it
    k = bars[4] + 1
    while not (ins[k][1] == "BRA" and not ins[k][3].startswith("@")):
        k += 1
    start = k + 1
    # per-tile prologue: from the back edge's target to the branch into the whole-tile body
    back = [k for k in range(bars[8], len(ins)) if ins[k][1] == "BRA" and ins[k][2] is not None and ins[k][2] < ins[k][0]
            and addr[bars[0]] < ins[k][2] < addr[bars[1]]]
    assert back, "no back edge of the tile loop"
    head = addr.index(ins[back[0]][2])
    into = [k for k in range(head, bars[1]) if ins[k][1] == "BRA" and ins[k][2] == ins[start][0]]
    assert into, "no branch into the whole-tile body"
    return {
        "prologue": range(head, into[0] + 1),
        "A": range(start, bars[5] + 1),
        "B": range(bars[5] + 1, bars[6] + 1),
        "C + deposit": range(bars[6] + 1, bars[7] + 1),
        "D": range(bars[7] + 1, bars[8] + 1),
        "epilogue": range(bars[8] + 1, back[0] + 1),
    }


def weights(ins, seg, name, trips):
    """Per-instruction weight inside one phase: the outermost loop counts `trips` times, loops nested in it 0 times."""
    w = {k: 1.0 for k in seg}
    if name not in ("C + deposit", "D"):
        return w
    addr = {ins[k][0]: k for k in seg}
    loops = [(addr[ins[k][2]], k) for k in seg if ins[k][1] == "BRA" and ins[k][2] in addr and ins[k][2] < ins[k][0]]
    if not loops:
        return w
    outer = max(loops, key=lambda l: l[1] - l[0])
    for k in range(outer[0], outer[1] + 1):
        w[k] = trips
    for lo, hi in loops:
        if (lo, hi) != outer:
            for k in range(lo, hi + 1):
                w[k] = 0.0
    return w


def model_trips():
    sys.path.insert(0, ROOT)
    import numpy as np
    from density_b200 import synth
    from tools import proto_tile_protocol_v6 as m6
    ntiles = 496
    q = synth.synth_text(ntiles * m6.TILE * 4).numpy().view(np.uint32)
    st = {}
    m6.flag_pass(q, stats=st)
    return float(np.ceil(np.array(st["warp_records"]) / 32).mean())


def table(sass, trips):
    ins = parse(sass)
    rows = collections.OrderedDict()
    for name, seg in cut(ins).items():
        w = weights(ins, seg, name, trips)
        c = collections.Counter()
        for k in seg:
            c[pipe(ins[k][1])] += w[k]
            c["static"] += 1
        rows[name] = c
    tot = collections.Counter()
    for c in rows.values():
        tot.update(c)
    rows["tile"] = tot
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--src", default=os.path.join(ROOT, "density_b200", "csrc", "chameleon_encode.cu"))
    ap.add_argument("--sass", help="cuobjdump -sass output to read instead of compiling --src")
    ap.add_argument("--trips", type=float, help="mean trips of the deposit and D loops per warp (default: from the model)")
    a = ap.parse_args()
    trips = a.trips if a.trips is not None else model_trips()
    sass = open(a.sass).read() if a.sass else sass_of(a.src)
    print(f"{a.sass or a.src}: weighted warp instructions per tile and warp (loop trips {trips:.3f})")
    print(f"| phase | static | {' | '.join(PIPES)} | weighted total |")
    print("|---|" + "---|" * (len(PIPES) + 2))
    for name, c in table(sass, trips).items():
        print(f"| {name} | {c['static']} | " + " | ".join(f"{c[p]:.0f}" for p in PIPES) + f" | {sum(c[p] for p in PIPES):.0f} |")


if __name__ == "__main__":
    main()
