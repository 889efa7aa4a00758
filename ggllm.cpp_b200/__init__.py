"""ggllm.cpp_b200 -- H100-native quantized-inference backend for Falcon (drop-in for the ggml_cuda_* surface).

The product is the C-ABI shared library ``csrc/libggml_b200.so`` (declared in ``include/ggml_b200.h``); this
package only holds its sources, the build recipe and thin ctypes bindings used by the tests and bench.py.
"""
