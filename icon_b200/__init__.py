"""icon_b200: sm_90a kernels + host mirror for ICON's occupancy-query / mesh-extraction hot path.

`import icon_b200` is light (no CUDA library needed); `icon_b200.ops` / `icon_b200._C` load
libicon_b200.so and raise ImportError if it has not been built (python -m icon_b200.build).
"""
__version__ = "0.1.0"
