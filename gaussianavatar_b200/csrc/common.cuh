// Shared helpers for libgavatar_sm90.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>

#include "../../include/gavatar.h"

namespace ga {

void set_error(const char *fmt, ...);
void count_launch(int n = 1);
// Optional per-kernel CUDA-event timing (bench.py's roofline leg): begin/end bracket one launch on its stream.
void prof_begin(cudaStream_t st);
void prof_end(const char *name, cudaStream_t st);
struct ProfScope {
    const char *name; cudaStream_t st;
    ProfScope(const char *n, cudaStream_t s) : name(n), st(s) { prof_begin(s); }
    ~ProfScope() { prof_end(name, st); }
};

#define GA_CHECK_CUDA(expr)                                                                          \
    do {                                                                                             \
        cudaError_t _e = (expr);                                                                     \
        if (_e != cudaSuccess) {                                                                     \
            ::ga::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return GA_ERR_CUDA;                                                                      \
        }                                                                                            \
    } while (0)

#define GA_CHECK_LAUNCH(name)                                                                        \
    do {                                                                                             \
        ::ga::count_launch();                                                                        \
        cudaError_t _e = cudaGetLastError();                                                         \
        if (_e != cudaSuccess) {                                                                     \
            ::ga::set_error("launch of %s failed: %s (%s:%d)", name, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return GA_ERR_CUDA;                                                                      \
        }                                                                                            \
    } while (0)

#define GA_REQUIRE(cond, ...)                                                                        \
    do {                                                                                             \
        if (!(cond)) {                                                                               \
            ::ga::set_error(__VA_ARGS__);                                                            \
            return GA_ERR_INVALID;                                                                   \
        }                                                                                            \
    } while (0)

constexpr size_t kAlign = 256;
inline size_t align_up(size_t x, size_t a = kAlign) { return (x + a - 1) / a * a; }

// Bump carving of a caller-owned byte buffer into aligned typed regions.
struct Carver {
    char *base;
    size_t off;
    explicit Carver(void *p) : base(static_cast<char *>(p)), off(0) {}
    template <typename T> T *take(size_t n)
    {
        off = align_up(off);
        T *r = reinterpret_cast<T *>(base + off);
        off += n * sizeof(T);
        return r;
    }
    size_t used() const { return align_up(off); }
};

inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// cudaFuncSetAttribute (opt-in to > 48 KB of dynamic shared memory) applies to the CURRENT device only: remember it per call site AND
// per device, so that a process that drives a second GPU does not launch with the default limit there.
struct PerDeviceOnce {
    bool done[64] = {};
    bool first()
    {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;      // unknown device: just set the attribute again
        if (done[dev]) return false;
        done[dev] = true;
        return true;
    }
};

constexpr int kNumSMs = 132;  // H100 SXM (compile-time grid constants of the heads / split-K kernels)
int num_sms();                // multiProcessorCount of the current device, queried once per device

// 16-byte vector reduction to global memory (sm_90+): one L2 atomic for four consecutive floats (16-byte aligned address)
__device__ __forceinline__ void red_add_v4(float *addr, float a, float b, float c, float d)
{
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
// the same for two consecutive floats (8-byte aligned address)
__device__ __forceinline__ void red_add_v2(float *addr, float a, float b)
{
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

}  // namespace ga
