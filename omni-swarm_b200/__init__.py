"""omniswarm_b200: H100-native loop-closure front-end + pose-graph back-end for Omni-swarm.

The product is the C-ABI shared library `csrc/libomniswarm_b200.so` (hand-written sm_90a CUDA);
the Python modules here are the thin host-side mirror of the reference's C++ call sites
(SuperPointTensorRT, MobileNetVLADTensorRT, faiss::IndexFlatIP, cv::BFMatcher,
SwarmLocalizationSolver::solve_once) used by the tests and by bench.py.
"""
__version__ = "0.1.0"
