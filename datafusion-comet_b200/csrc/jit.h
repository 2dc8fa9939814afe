// jit.h -- NVRTC compilation of generated pipeline kernels for sm_90a + module cache.
#pragma once
#include "codegen.h"

#include <cuda_runtime.h>
#include <map>
#include <mutex>
#include <memory>
#include <string>
#include <vector>

namespace cb200 {

struct CompiledModule {
    std::vector<char> cubin;
    cudaLibrary_t lib = nullptr;
    std::map<std::string, cudaKernel_t> kernels;
    std::mutex mu; // modules are shared by every plan (and task thread) that uses the same pipeline
    bool loaded = false;
    ~CompiledModule();
    cudaKernel_t kernel(const std::string& name);
};

struct JitError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

// Compile (or fetch from the in-memory / on-disk cache) the module for `g`.  With load=false the
// cubin is produced but not loaded on a device (works on a CPU-only box: NVRTC needs no GPU).
std::shared_ptr<CompiledModule> jit_get(const GeneratedKernel& g, bool load);
// On-disk cubin caches, searched in order: CB200_CACHE_DIR when it is set, then `.jitcache` next to the
// library (filled by the build).  New cubins are written to the first, so a process whose install tree is
// read-only (or must stay unchanged) points CB200_CACHE_DIR at a writable directory and still finds the
// cubins the build shipped.
std::vector<std::string> jit_cache_dirs();

} // namespace cb200
