"""asyrp_official_b200 — Asyrp sampling engine for the H100 (DDIM reverse loop + UNet forward).

The compute path is libasyrp_b200.so (hand-written sm_90a CUDA behind a C ABI, include/asyrp_b200.h);
this package is the host-side mirror of the reference's Python entry points for that path.
"""
__version__ = "0.1.0"
