"""H100-native batched multirotor simulator: drop-in for the two hot paths of
ntnu-arl/aerial_gym_simulator (dynamics+controller step, ray-cast sensors).

The compute path is hand-written sm_90a CUDA behind the C ABI in
``include/aerial_gym_b200.h``; this package is the host-side mirror of the
reference's Python surface.  There is no CPU fallback: importing the native
layer without the built library, or calling it without a CUDA device, raises."""

__version__ = "0.1.0"
