"""regenie_b200 -- H100-native hot path of regenie Step 1 / Step 2.

The product is the C ABI in include/rg_b200.h (librg_b200.so, hand-written sm_90a kernels)
and the C++ host driver `rgb200`; this package only holds the build recipe, a ctypes binding
used by tests/bench, and the synthetic-panel generator.
"""
__all__ = ["capi", "build", "synth"]
