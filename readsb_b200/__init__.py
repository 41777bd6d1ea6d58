"""readsb_b200 — Hopper-native Mode-S demodulator behind readsb's demodulate2400() boundary.

Only the hot path lives here: `csrc/` (CUDA kernels + the C ABI declared in include/b200_demod.h),
`demod.py` (host-side mirror of the reference interface over that C ABI), `synth/` (synthetic
capture generator) and `build.py`.  There is no CPU implementation of the demodulator in this
package: importing `readsb_b200.demod` without the built CUDA library raises.
"""
__version__ = "0.1.0"
