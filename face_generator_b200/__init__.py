"""face_generator_b200 -- H100-native GAN train-step hot path of aleju/face-generator.

The product is `libfg_b200.so` (hand-written sm_90a CUDA behind the C ABI in include/fg_b200.h).
This Python package is only the host-side mirror of the reference's Lua plugin surface
(nn.Module-style G/D objects, BCECriterion, interruptableAdam, the adversarial.train loop body) used by
tests and bench.py; the reference-side binding is the LuaJIT FFI shim under face_generator_b200/lua/.
There is NO CPU fallback: importing works anywhere, but every compute call needs an H100 (sm_90).
"""
from .lib import FGError, load_library, Context, C2f, S16, hyper_default, MASK_PER_SAMPLE, NOISE_DIM  # noqa: F401
from . import nn, adversarial, adversarial_c2f  # noqa: F401
