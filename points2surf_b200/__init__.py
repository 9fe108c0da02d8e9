"""points2surf_b200 -- H100-native Points2Surf SDF-inference hot path.

Host-side mirror (Python, like the reference) of the reference's interface for the
path SURVEY.md section 8 names, on top of the C-ABI library `libp2s_b200.so`
(include/p2s_b200.h) which holds the hand-written sm_90a CUDA kernels.
There is no CPU fallback: importing `points2surf_b200._lib` raises if the library
has not been built, and every op raises if CUDA is unavailable.
"""
__version__ = '0.1.0'
