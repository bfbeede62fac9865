"""beast-mcmc_b200: an H100-native (sm_90a) tree-likelihood engine that sits behind BEAST's
BEAGLE boundary (libhmsbeagle C ABI + libhmsbeagle-jni JNI shim).

The directory name carries a hyphen (as the project is named); import it as
``beast_mcmc_b200`` through the loader shim ``beast_mcmc_b200.py`` at the repo root.

  csrc/                  CUDA kernels, the C ABI (include/libhmsbeagle_b200.h) and the JNI shim
  beagle.py              ctypes mirror of the ``beagle.Beagle`` Java interface over the C ABI
  build.py               in-tree nvcc build of the shared libraries

The Python re-enactments of the reference's Java callers (test/bench harness) live in ``harness/`` at the repo root,
not here: the product is the two shared libraries under csrc/.
"""
__all__ = ["beagle", "build"]
