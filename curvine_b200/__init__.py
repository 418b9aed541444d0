"""curvine_b200: GPU-native (H100, sm_90a) sequential block-read path for Curvine (see DESIGN.md).

The package is a thin Python mirror over libcurvine_b200.so's C ABI (include/*.h);
importing it never falls back to a CPU implementation.
"""
__version__ = "0.1.0"
