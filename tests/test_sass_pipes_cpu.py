"""tools/sass_pipes.py finds the whole-tile path of the flag pass in the compiled kernel, and the model's records per warp add up to its
records per tile. Needs nvcc and cuobjdump, no GPU."""
import os
import shutil

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_model_records_per_warp_add_up():
    from tools import proto_tile_protocol_v6 as m6
    d = np.fromfile(os.path.join(ROOT, "tests", "golden", "dickens_200k.bin"), np.uint8)
    q = d[:160000].view(np.uint32).copy()
    st = {}
    m6.flag_pass(q, stats=st)
    w = np.array(st["warp_records"])
    assert w.shape == (st["tiles"], m6.TILE // m6.REGION)
    assert int(w.sum()) == st["dirty"]


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_sass_pipes_cuts_the_whole_tile_path():
    from tools import sass_pipes
    rows = sass_pipes.table(sass_pipes.sass_of(os.path.join(ROOT, "density_b200", "csrc", "chameleon_encode.cu")), trips=1.0)
    for phase in ("prologue", "A", "B", "C + deposit", "D", "epilogue"):
        assert rows[phase]["static"] > 0, phase
    assert rows["tile"]["static"] == sum(rows[p]["static"] for p in rows if p != "tile")
    assert rows["C + deposit"]["MIO"] > 0 and rows["A"]["FMA"] > 0
