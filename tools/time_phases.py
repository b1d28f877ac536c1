"""Per-phase cycle counts of cham_flag_pass6 (needs a lib built with -DDNS_PHASE_TIMING: tools/build_variant.sh timing "-DDNS_PHASE_TIMING";
run with DENSITY_B200_SO=density_b200/_variants/lib_timing.so)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import density_b200
from density_b200 import synth
n = 1 << 30
d_in = synth.synth_text(n, device="cuda")
d_out = torch.empty(density_b200.Chameleon.safe_encode_buffer_size(n), dtype=torch.uint8, device="cuda")
d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
for _ in range(2):
    density_b200.encode_device("chameleon", d_in, d_out, d_sz)
torch.cuda.synchronize()
print("out", int(d_sz.item()))
