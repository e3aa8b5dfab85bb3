// Process-wide plumbing of the C ABI: error string, version, launch counter.
#include <atomic>
#include <cstdarg>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "common.cuh"

namespace ga {
namespace {
thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};
}  // namespace

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int num_sms()
{
    static int cached[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return kNumSMs;
    if (cached[dev] == 0) {
        int n = 0;
        cached[dev] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : kNumSMs;
    }
    return cached[dev];
}

// ---- per-kernel event timing ----------------------------------------------------------------------------------------
namespace {
struct ProfRec { const char *name; cudaEvent_t a, b; };
bool g_prof_on = false;
std::vector<ProfRec> g_prof;
std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_pool;
cudaEvent_t g_cur_a = nullptr, g_cur_b = nullptr;
}  // namespace

void prof_begin(cudaStream_t st)
{
    if (!g_prof_on) return;
    if (g_pool.empty()) {
        cudaEvent_t a, b;
        cudaEventCreate(&a); cudaEventCreate(&b);
        g_cur_a = a; g_cur_b = b;
    } else { g_cur_a = g_pool.back().first; g_cur_b = g_pool.back().second; g_pool.pop_back(); }
    cudaEventRecord(g_cur_a, st);
}
void prof_end(const char *name, cudaStream_t st)
{
    if (!g_prof_on || !g_cur_a) return;
    cudaEventRecord(g_cur_b, st);
    g_prof.push_back(ProfRec{name, g_cur_a, g_cur_b});
    g_cur_a = g_cur_b = nullptr;
}
}  // namespace ga

extern "C" void ga_profile_enable(int on) { ga::g_prof_on = on != 0; }
// Synchronises the device, then writes "name count total_ms\n" lines (aggregated per kernel name) and clears the log.
extern "C" int ga_profile_report(char *buf, size_t cap)
{
    cudaDeviceSynchronize();
    std::map<std::string, std::pair<long long, double>> agg;
    for (auto &r : ga::g_prof) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, r.a, r.b);
        auto &e = agg[r.name];
        e.first += 1; e.second += ms;
        ga::g_pool.emplace_back(r.a, r.b);
    }
    ga::g_prof.clear();
    size_t off = 0;
    if (buf && cap) buf[0] = 0;
    for (auto &kv : agg) {
        int n = snprintf(buf + off, off < cap ? cap - off : 0, "%s %lld %.6f\n", kv.first.c_str(), kv.second.first, kv.second.second);
        if (n < 0 || off + (size_t)n >= cap) return GA_ERR_CAPACITY;
        off += (size_t)n;
    }
    return GA_OK;
}

extern "C" int ga_version(void) { return 110; }
extern "C" const char *ga_last_error(void) { return ga::g_err; }
extern "C" long long ga_launch_count(void) { return ga::g_launches.load(std::memory_order_relaxed); }
