"""catgrasp_b200 -- H100-native grasp-scoring hot path of CaTGrasp (see DESIGN.md).

Importing the package is cheap and GPU-free; every compute entry point goes through
libcatgrasp_b200.so (hand-written sm_90a CUDA) and raises if it is missing.
"""
__version__ = "0.1.0"
