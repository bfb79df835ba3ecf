// TEST INFRASTRUCTURE: the one translation unit of the emulated libfplgpu that owns the emulator's state — the fiber scheduler
// (emu_cuda_impl.h), the cp.async / mbarrier emulation, and NVRTC + the three driver calls fpl_jit.cu makes, where "compiling"
// a kernel means building its source for the host with g++ behind the emulator and "loading the cubin" means dlopen.
#include "emu_cuda_impl.h"
#include "fake/cuda.h"
#include "fake/nvrtc.h"
#include <dlfcn.h>
#include <map>
#include <mutex>
#include <string>

// ---------------- cp.async: completion at the latest legal moment (default) or at issue ----------------
namespace emu {
namespace {
int cp_lazy = 1;
struct Copy { uint8_t* dst; const uint8_t* src; int n, size; };
struct Queue { unsigned long long serial = 0; std::vector<Copy> open; std::vector<std::vector<Copy>> groups; };
Queue queues[1024];
Queue& q() { Queue& x = queues[tid_in_block()]; if (x.serial != block_serial) { x.serial = block_serial; x.open.clear(); x.groups.clear(); } return x; }
void now(const Copy& c) { if (c.n > 0) memcpy(c.dst, c.src, c.n); memset(c.dst + c.n, 0, c.size - c.n); }
struct Mbar { uint32_t phase; int32_t pending; };       // pending: bytes still to arrive, +2^30 while the arrival is outstanding
void settle(Mbar* m) { if (m->pending == 0) { m->phase++; m->pending = 1 << 30; note_progress(); } }
}  // namespace
void cp_async(uint32_t dst, const void* src, int n, int size) {
    Copy c = {(uint8_t*)from_shared(dst), (const uint8_t*)src, n, size};
    if (cp_lazy) q().open.push_back(c); else now(c);
}
void cp_commit() { if (cp_lazy) { Queue& x = q(); x.groups.push_back(x.open); x.open.clear(); } }
void cp_wait(int n_pending) {
    if (!cp_lazy) return;
    Queue& x = q();
    while ((int)x.groups.size() > n_pending) { for (const Copy& c : x.groups.front()) now(c); x.groups.erase(x.groups.begin()); }
}
void mbar_init(uint32_t bar) { Mbar* m = (Mbar*)from_shared(bar); m->phase = 0; m->pending = 1 << 30; }
void mbar_expect(uint32_t bar, uint32_t bytes) { Mbar* m = (Mbar*)from_shared(bar); m->pending += (int32_t)bytes - (1 << 30); settle(m); }
void mbar_wait(uint32_t bar, uint32_t parity) { Mbar* m = (Mbar*)from_shared(bar); while ((m->phase & 1u) == parity) yield(); }
void bulk(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    memcpy(from_shared(dst), src, bytes);
    Mbar* m = (Mbar*)from_shared(bar); m->pending -= (int32_t)bytes; settle(m);
}
}  // namespace emu
extern "C" void emu_set_cp_async_lazy(int on) { emu::cp_lazy = on; }
extern "C" long long emu_collectives() { return emu::collectives; }
namespace emu { long long live_allocs = 0, fail_alloc_in = 0; }      // fake/cuda_runtime.h: emu_alloc
extern "C" long long emu_live_allocs() { return emu::live_allocs; }
// -> the count it replaces: > 0 when the allocation it was set for never came
extern "C" long long emu_fail_alloc(long long k) { const long long was = emu::fail_alloc_in; emu::fail_alloc_in = k; return was; }
extern "C" long long emu_blocks() { return (long long)emu::block_serial; }
// kernel name ("k_trim" of "k_trim<1>(P, b, ...)", "k_scan_jit" of "jit::k_scan_jit(...)") -> launches so far
namespace emu { namespace { std::mutex launch_count_mu; std::map<std::string, long long> launch_count; } }
void emu::note_launch(const char* call) {
    std::string name(call);
    name = name.substr(0, name.find_first_of("<( "));
    if (name.rfind("::") != std::string::npos) name = name.substr(name.rfind("::") + 2);
    std::lock_guard<std::mutex> lock(launch_count_mu);
    launch_count[name]++;
}
// -> the launches so far of the kernels whose names start with prefix ("": all)
extern "C" long long emu_launches(const char* prefix) {
    std::lock_guard<std::mutex> lock(emu::launch_count_mu);
    long long n = 0;
    for (const auto& kv : emu::launch_count)
        if (kv.first.compare(0, strlen(prefix), prefix) == 0) n += kv.second;
    return n;
}

// ---------------- streams and events (fake/cuda_runtime.h): ids never reused; the live ones, an event with its timestamp ----------------
namespace emu {
namespace {
std::mutex handle_mu;                   // host threads with a context each create and destroy their own
std::map<const void*, double> handles;
uintptr_t last_handle = 0x100000;
long long fail_handle_in = 0, bad_handles = 0, failed_kind = 0;
}  // namespace
void* handle_new(int kind) {
    std::lock_guard<std::mutex> lock(handle_mu);
    if (fail_handle_in > 0 && --fail_handle_in == 0) { failed_kind = kind; return nullptr; }
    last_handle += 16;
    handles[(const void*)last_handle] = 0;
    return (void*)last_handle;
}
double* handle(const void* h) {
    std::lock_guard<std::mutex> lock(handle_mu);
    auto it = handles.find(h);
    if (it == handles.end()) { bad_handles++; return nullptr; }
    return &it->second;
}
bool handle_free(const void* h) {
    std::lock_guard<std::mutex> lock(handle_mu);
    if (handles.erase(h)) return true;
    bad_handles++;
    return false;
}
}  // namespace emu
extern "C" long long emu_live_handles() { std::lock_guard<std::mutex> lock(emu::handle_mu); return (long long)emu::handles.size(); }
extern "C" long long emu_bad_handles() { std::lock_guard<std::mutex> lock(emu::handle_mu); return emu::bad_handles; }
// -> the count it replaces: > 0 when the creation it was set for never came
extern "C" long long emu_fail_handle(long long k) {
    std::lock_guard<std::mutex> lock(emu::handle_mu);
    const long long was = emu::fail_handle_in;
    emu::fail_handle_in = k;
    return was;
}
// -> what the creation that emu_fail_handle made fail created (EMU_STREAM, EMU_EVENT, EMU_TIMING_EVENT; 0: none), and forgets it
extern "C" long long emu_failed_handle_kind() {
    std::lock_guard<std::mutex> lock(emu::handle_mu);
    const long long k = emu::failed_kind;
    emu::failed_kind = 0;
    return k;
}

// ---------------- NVRTC + driver: kernels "compiled" for the host ----------------
struct EmuNvrtcProgram { std::string src, log, so; };
static std::mutex jit_mu;
extern "C" {
nvrtcResult nvrtcCreateProgram(nvrtcProgram* prog, const char* src, const char*, int, const char* const*, const char* const*) {
    *prog = new EmuNvrtcProgram();
    (*prog)->src = src;
    return NVRTC_SUCCESS;
}
nvrtcResult nvrtcDestroyProgram(nvrtcProgram* prog) { delete *prog; *prog = nullptr; return NVRTC_SUCCESS; }
nvrtcResult nvrtcCompileProgram(nvrtcProgram p, int, const char* const*) {
    std::lock_guard<std::mutex> lock(jit_mu);
    unsigned long long h = 1469598103934665603ull;
    for (unsigned char ch : p->src) h = (h ^ ch) * 1099511628211ull;
    char base[256];
    snprintf(base, sizeof(base), "/tmp/fpl_emu_jit_%016llx_%s", h, EMU_BUILD_TAG);
    p->so = std::string(base) + ".so";
    if (FILE* f = fopen(p->so.c_str(), "rb")) { fclose(f); return NVRTC_SUCCESS; }
    const std::string cpp = std::string(base) + ".cpp";
    FILE* f = fopen(cpp.c_str(), "w");
    if (!f) { p->log = "cannot write " + cpp; return 1; }
    fputs("#include \"emu_cuda.h\"\nnamespace jit {\n", f);
    fputs(p->src.c_str(), f);
    fputs("\n}  // namespace jit\n"
          "extern \"C\" void jit_scan(unsigned grid, unsigned block, unsigned smem, const uint8_t* seq, const uint8_t* qual, const int64_t* offsets,\n"
          "                         void* st, int64_t n, unsigned one) {\n"
          "    EMU_LAUNCH((grid), (block), (smem), jit::k_scan_jit(seq, qual, (const jit::int64_t*)offsets, (jit::ReadState*)st, (jit::int64_t)n, one));\n"
          "}\n", f);
    fclose(f);
    const std::string tmp = p->so + ".tmp";
    const std::string cmd = std::string("g++ -std=c++17 -O1 -fPIC -shared -w -I ") + EMU_SIMT_DIR + " -o " + tmp + " " + cpp + " " + EMU_LIB_PATH +
                            " -Wl,-rpath," + EMU_LIB_DIR + " > " + base + ".log 2>&1 && mv " + tmp + " " + p->so;
    if (system(cmd.c_str()) != 0) { p->log = "g++ failed: see " + std::string(base) + ".log"; return 1; }
    return NVRTC_SUCCESS;
}
nvrtcResult nvrtcGetProgramLogSize(nvrtcProgram p, size_t* n) { *n = p->log.size() + 1; return NVRTC_SUCCESS; }
nvrtcResult nvrtcGetProgramLog(nvrtcProgram p, char* log) { memcpy(log, p->log.c_str(), p->log.size() + 1); return NVRTC_SUCCESS; }
nvrtcResult nvrtcGetCUBINSize(nvrtcProgram p, size_t* n) { *n = p->so.size() + 1; return NVRTC_SUCCESS; }
nvrtcResult nvrtcGetCUBIN(nvrtcProgram p, char* cubin) { memcpy(cubin, p->so.c_str(), p->so.size() + 1); return NVRTC_SUCCESS; }
const char* nvrtcGetErrorString(nvrtcResult r) { return r == NVRTC_SUCCESS ? "NVRTC_SUCCESS" : "emulated NVRTC: host compile failed"; }

CUresult cuModuleLoadData(CUmodule* mod, const void* image) { *mod = dlopen((const char*)image, RTLD_NOW | RTLD_LOCAL); return *mod ? CUDA_SUCCESS : 200; }
CUresult cuModuleGetFunction(CUfunction* fn, CUmodule mod, const char*) { *fn = dlsym(mod, "jit_scan"); return *fn ? CUDA_SUCCESS : 500; }
CUresult cuLaunchKernel(CUfunction f, unsigned gx, unsigned, unsigned, unsigned bx, unsigned, unsigned, unsigned smem, CUstream, void** args, void**) {
    typedef void (*fn_t)(unsigned, unsigned, unsigned, const uint8_t*, const uint8_t*, const int64_t*, void*, int64_t, unsigned);
    ((fn_t)f)(gx, bx, smem, *(const uint8_t**)args[0], *(const uint8_t**)args[1], *(const int64_t**)args[2], *(void**)args[3], *(int64_t*)args[4],
              *(unsigned*)args[5]);
    return CUDA_SUCCESS;
}
CUresult cuGetErrorString(CUresult, const char** s) { *s = "emulated driver error"; return CUDA_SUCCESS; }
}
