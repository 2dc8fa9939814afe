// jit.cpp -- NVRTC -> sm_90a cubin -> cudaLibraryLoadData.  The device library and the kernel
// skeletons (device/cb_math.h, device/cb_kernels.cuh) are embedded in the .so as strings
// (device_src.inc, generated at build time) and handed to NVRTC as in-memory headers.
#include "jit.h"

#include <dlfcn.h>
#include <nvrtc.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <mutex>

namespace cb200 {

extern const char* const cb_math_src;
extern const char* const cb_params_src;
extern const char* const cb_kernels_src;

CompiledModule::~CompiledModule() {
    if (lib) cudaLibraryUnload(lib);
}

cudaKernel_t CompiledModule::kernel(const std::string& name) {
    std::lock_guard<std::mutex> lk(mu);
    auto it = kernels.find(name);
    if (it != kernels.end()) return it->second;
    cudaKernel_t k = nullptr;
    cudaError_t e = cudaLibraryGetKernel(&k, lib, name.c_str());
    if (e != cudaSuccess) throw JitError("cudaLibraryGetKernel(" + name + "): " + cudaGetErrorString(e));
    kernels[name] = k;
    return k;
}

std::vector<std::string> jit_cache_dirs() {
    std::vector<std::string> dirs;
    const char* env = getenv("CB200_CACHE_DIR");
    if (env && *env) dirs.push_back(env);
    Dl_info info;
    if (dladdr((void*)&jit_cache_dirs, &info) && info.dli_fname) {
        std::string p = info.dli_fname;
        size_t s = p.rfind('/');
        dirs.push_back((s == std::string::npos ? std::string(".") : p.substr(0, s)) + "/.jitcache");
    }
    if (dirs.empty()) dirs.push_back("/tmp/cb200_jitcache");
    return dirs;
}

// --fmad=false: every float expression node rounds once, like the reference's per-node arrays
static const char* const kNvrtcOpts[] = {"--gpu-architecture=sm_90a", "-std=c++17", "-lineinfo", "--fmad=false"};

// cubins depend on the device headers and the compile options (the target architecture above all) as much as on
// the generated translation unit
static std::string headers_tag() {
    static std::string tag;
    if (tag.empty()) {
        uint64_t h = 1469598103934665603ull;
        for (const char* src : {cb_math_src, cb_params_src, cb_kernels_src})
            for (const char* c = src; *c; c++) { h ^= (unsigned char)*c; h *= 1099511628211ull; }
        for (const char* opt : kNvrtcOpts)
            for (const char* c = opt; *c; c++) { h ^= (unsigned char)*c; h *= 1099511628211ull; }
        char buf[32];
        snprintf(buf, sizeof(buf), "%016llx", (unsigned long long)h);
        tag = buf;
    }
    return tag;
}

static std::mutex g_mu;
static std::map<std::string, std::shared_ptr<CompiledModule>> g_cache;

static std::vector<char> compile(const GeneratedKernel& g) {
    nvrtcProgram prog;
    const char* headers[3] = {cb_math_src, cb_params_src, cb_kernels_src};
    const char* names[3] = {"cb_math.h", "cb_params.h", "cb_kernels.cuh"};
    if (nvrtcCreateProgram(&prog, g.source.c_str(), ("cb200_" + g.key + ".cu").c_str(), 3, headers, names) != NVRTC_SUCCESS)
        throw JitError("nvrtcCreateProgram failed");
    nvrtcResult r = nvrtcCompileProgram(prog, (int)(sizeof(kNvrtcOpts) / sizeof(kNvrtcOpts[0])), kNvrtcOpts);
    if (r != NVRTC_SUCCESS) {
        size_t n = 0;
        nvrtcGetProgramLogSize(prog, &n);
        std::string log(n, '\0');
        nvrtcGetProgramLog(prog, &log[0]);
        nvrtcDestroyProgram(&prog);
        throw JitError("NVRTC compile failed for pipeline " + g.key + ":\n" + log);
    }
    size_t n = 0;
    if (nvrtcGetCUBINSize(prog, &n) != NVRTC_SUCCESS || n == 0) {
        nvrtcDestroyProgram(&prog);
        throw JitError("NVRTC produced no cubin (sm_90a not supported by this NVRTC?)");
    }
    std::vector<char> cubin(n);
    nvrtcGetCUBIN(prog, cubin.data());
    nvrtcDestroyProgram(&prog);
    return cubin;
}

std::shared_ptr<CompiledModule> jit_get(const GeneratedKernel& g, bool load) {
    std::lock_guard<std::mutex> lk(g_mu);
    std::shared_ptr<CompiledModule> m;
    auto it = g_cache.find(g.key);
    if (it != g_cache.end()) m = it->second;
    if (!m) {
        m = std::make_shared<CompiledModule>();
        const std::vector<std::string> dirs = jit_cache_dirs();
        const std::string file = "/" + g.key + "_" + headers_tag() + ".cubin";
        for (const std::string& d : dirs) {
            std::ifstream in(d + file, std::ios::binary);
            if (in) m->cubin.assign(std::istreambuf_iterator<char>(in), std::istreambuf_iterator<char>());
            if (!m->cubin.empty()) break;
        }
        if (m->cubin.empty()) {
            const std::string& dir = dirs.front();
            const std::string path = dir + file;
            m->cubin = compile(g);
            mkdir(dir.c_str(), 0755);
            std::string tmp = path + ".tmp" + std::to_string((long)getpid());
            std::ofstream out(tmp, std::ios::binary);
            if (out) {
                out.write(m->cubin.data(), (std::streamsize)m->cubin.size());
                out.close();
                rename(tmp.c_str(), path.c_str());
                if (getenv("CB200_DUMP_SRC")) {
                    std::ofstream src(dir + "/" + g.key + ".cu");
                    src << g.source;
                }
            }
        }
        g_cache[g.key] = m;
    }
    if (load && !m->loaded) {
        cudaError_t e = cudaLibraryLoadData(&m->lib, m->cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
        if (e != cudaSuccess) throw JitError(std::string("cudaLibraryLoadData: ") + cudaGetErrorString(e));
        m->loaded = true;
    }
    return m;
}

} // namespace cb200
