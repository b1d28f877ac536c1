"""density_b200 — H100-native (sm_90a) Chameleon / Cheetah / Lion encode/decode hot path of g1mv/density.

The product is libdensity_b200.so (hand-written CUDA behind the reference's own C ABI, include/density_b200.h);
this package is the thin host-side mirror of the reference's `Codec` interface plus the torch.distributed plumbing
for the sharded multi-GPU path.
"""
from .codec import (CODECS, Chameleon, Cheetah, DecodeError, EncodeError, Lion, decode_device, decode_range_device,  # noqa: F401
                    decode_range_indexed_device, decoded_size_device, encode_device, index_build_device)
from ._lib import DensityB200Error, SO_PATH, load  # noqa: F401

__version__ = "0.1.0"
