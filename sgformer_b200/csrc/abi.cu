// Library-level C-ABI entry points (version string, launch counter).
#include <cuda_runtime.h>
#include "launch_count.h"
#include "../../include/sgformer_b200.h"

namespace sgf {
std::atomic<int64_t> g_launches{0};
}

extern "C" const char* sgf_version(void) { return "sgformer_b200 0.1.0 sm_90a"; }
extern "C" int64_t sgf_launch_count(void) { return sgf::g_launches.load(std::memory_order_relaxed); }

// This library links its own (static) CUDA runtime; the host framework selects the device on its runtime, so the
// Python layer forwards the choice before the first launch on a thread / after every change.
extern "C" int sgf_set_device(int device) { return (int)cudaSetDevice(device); }
