"""go-snark-study_b200 — H100-native Groth16 / Pinocchio prove path.

Host-side mirror of the reference's Go package API for the prove path
(bn128.G1/G2, r1csqap.PolynomialField, groth16.GenerateProofs,
snark.GenerateProofs) over the C ABI of ``lib/libb200snark.so``
(include/b200snark.h).  There is no CPU fallback: importing ``_lib`` without
the built CUDA library, or calling it without a GPU, raises.
"""
__version__ = "0.1.0"
