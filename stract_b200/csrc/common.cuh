// common.cuh -- shared helpers of libstract_b200 (error plumbing, launch accounting, small device utils)
#pragma once
#ifndef SB200_EMU   // tests/emu builds the same sources for a CPU SIMT emulator and force-includes its own shim
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#endif
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <string.h>
#include <atomic>
#include <new>

#include "../../include/stract_b200.h"

namespace sb200 {

// ---- error plumbing: nothing throws across the C ABI ---------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

struct Err {
  int code;
};

#define SB_CUDA(expr)                                                                   \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      ::sb200::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,           \
                         cudaGetErrorString(_e));                                       \
      return (_e == cudaErrorMemoryAllocation) ? SB200_ENOMEM : SB200_ECUDA;            \
    }                                                                                   \
  } while (0)

#define SB_TRY(expr)           \
  do {                         \
    int _r = (expr);           \
    if (_r != SB200_OK) return _r; \
  } while (0)

#define SB_FAIL(code, ...)            \
  do {                                \
    ::sb200::set_error(__VA_ARGS__);  \
    return (code);                    \
  } while (0)

// every kernel launch goes through this so gpu_launches in bench.py is a counted number
#ifndef SB200_EMU
#define SB_LAUNCH(kernel, grid, block, smem, stream, ...)                 \
  do {                                                                    \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);           \
    ::sb200::g_launches.fetch_add(1, std::memory_order_relaxed);          \
  } while (0)
// dynamic shared memory of a kernel
#define SB_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif

#define SB_CHECK_LAUNCH() SB_CUDA(cudaGetLastError())

// NVTX ranges around the host-visible phases (graph staging steps, HyperBall iterations, BM25 batches): they cost a
// few ns without a tool attached and give nsys / ncu timelines the reference's phase names (SURVEY section 5: the reference
// wraps the same phases in `tracing` spans).  Header-only NVTX v3, no extra library.
#ifndef SB200_EMU
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};
#else
struct NvtxRange { explicit NvtxRange(const char*) {} };
#endif

extern thread_local cudaStream_t t_pool_stream;
// opt-in slab arena (arena.h / arena.cu, SB200_ARENA=1): replaces cudaMallocAsync inside a PoolScope
bool arena_enabled();
void* arena_alloc(size_t bytes, cudaStream_t stream, int* dev_out);
void arena_free(void* p, cudaStream_t stream, int dev);
void arena_retire_stream(int dev, cudaStream_t stream);
struct PoolScope {
  cudaStream_t prev;
  explicit PoolScope(cudaStream_t s) : prev(t_pool_stream) { t_pool_stream = s; }
  ~PoolScope() { t_pool_stream = prev; }
};

// RAII device buffer (cudaMalloc or, inside a PoolScope, cudaMallocAsync); move-only
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  cudaStream_t pool_stream = nullptr;  // non-null: stream-ordered allocation (cudaMallocAsync) on that stream
  bool borrowed = false;               // caller-owned memory (sb200_hyperball_bind_state): never freed here
  int arena_dev = -1;                  // >= 0: block of that device's slab arena, "freed on" pool_stream
  DevBuf() {}
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n), pool_stream(o.pool_stream), borrowed(o.borrowed), arena_dev(o.arena_dev) {
    o.p = nullptr; o.n = 0; o.pool_stream = nullptr; o.borrowed = false; o.arena_dev = -1;
  }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      release(); p = o.p; n = o.n; pool_stream = o.pool_stream; borrowed = o.borrowed; arena_dev = o.arena_dev;
      o.p = nullptr; o.n = 0; o.pool_stream = nullptr; o.borrowed = false; o.arena_dev = -1;
    }
    return *this;
  }
  ~DevBuf() { release(); }
  void release() {
    if (p && !borrowed) {
      if (arena_dev >= 0) arena_free(p, pool_stream, arena_dev);
      else if (pool_stream) cudaFreeAsync(p, pool_stream);
      else cudaFree(p);
    }
    p = nullptr; n = 0; pool_stream = nullptr; borrowed = false; arena_dev = -1;
  }
  void adopt(T* ptr, size_t count) { release(); p = ptr; n = count; borrowed = true; }
  // Inside a PoolScope the buffer comes from the device's stream-ordered memory pool: the staging pipeline
  // allocates and frees tens of GB of temporaries per graph, and cudaMalloc/cudaFree of such sizes are slow;
  // pooled memory is recycled across creates.
  int alloc(size_t count) {
    release();
    if (count == 0) { n = 0; return SB200_OK; }
    cudaError_t e;
    if (t_pool_stream && arena_enabled() && (p = (T*)arena_alloc(count * sizeof(T), t_pool_stream, &arena_dev)) != nullptr) {
      pool_stream = t_pool_stream; n = count; return SB200_OK;
    }
    if (t_pool_stream) { e = cudaMallocAsync((void**)&p, count * sizeof(T), t_pool_stream); pool_stream = t_pool_stream; }
    else e = cudaMalloc((void**)&p, count * sizeof(T));
    if (e != cudaSuccess) {
      p = nullptr; pool_stream = nullptr;
      set_error("device allocation of %zu bytes failed: %s", count * sizeof(T), cudaGetErrorString(e));
      cudaGetLastError();
      return SB200_ENOMEM;
    }
    n = count;
    return SB200_OK;
  }
  size_t bytes() const { return n * sizeof(T); }
};

// copies `bytes` from a host-or-device pointer into device memory on `stream`
int copy_in(void* dst_dev, const void* src_any, size_t bytes, cudaStream_t stream);
bool is_device_ptr(const void* p);

static inline unsigned div_up(uint64_t a, uint64_t b) { return (unsigned)((a + b - 1) / b); }
// switch from the environment: unset -> dflt, "0"/"" -> off, anything else -> on
static inline bool env_flag(const char* name, bool dflt) {
  const char* e = getenv(name);
  if (!e) return dflt;
  return *e && *e != '0';
}

// ---- device helpers --------------------------------------------------------------------------
// Byte-wise unsigned max of 4 packed bytes, valid when every byte is < 128 -- which holds for HyperLogLog<64>
// registers (rho <= 65, hyperloglog.rs:4385-4396).  sm_90a has no SIMD byte max (`__vmaxu4` is emulated with
// 6 LOP3/SHF/PRMT/IADD, and the pull kernels issue one per 4 register bytes gathered), so use 3 instructions:
//   d = a + 0x80808080 - b   no carry/borrow crosses a byte (a_i + 0x80 <= 0xFF and >= 0x80 > b_i); MSB_i = (a_i >= b_i)
//   m = PRMT sign-replicate  0xFF where a_i >= b_i, else 0x00
//   r = (a & m) | (b & ~m)   one LOP3
__device__ __forceinline__ uint32_t bmax4_7bit(uint32_t a, uint32_t b) {
  const uint32_t d = a + 0x80808080u - b;
  uint32_t m;
  // generic-mode PRMT: a selector nibble with its msb set replicates the SIGN of the selected byte over the byte
  // (the `__byte_perm` intrinsic masks that bit off, hence the inline PTX)
#ifndef SB200_EMU
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(m) : "r"(d), "r"(0u), "r"(0xba98u));
#else
  m = ((d >> 7) & 0x01010101u) * 0xFFu;   // what that PRMT computes (tests/emu)
#endif
  return (a & m) | (b & ~m);
}
__device__ __forceinline__ uint4 vmax_u8x16(uint4 a, uint4 b) {
  return make_uint4(bmax4_7bit(a.x, b.x), bmax4_7bit(a.y, b.y), bmax4_7bit(a.z, b.z), bmax4_7bit(a.w, b.w));
}
__device__ __forceinline__ bool ne_u4(uint4 a, uint4 b) {
  return ((a.x ^ b.x) | (a.y ^ b.y) | (a.z ^ b.z) | (a.w ^ b.w)) != 0u;
}

// streaming (read-once) load: do not allocate in L1
__device__ __forceinline__ uint32_t ld_stream_u32(const uint32_t* p) {
#ifndef SB200_EMU
  uint32_t v;
  asm volatile("ld.global.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
#else
  return *p;
#endif
}

// 16-B loads of data that no thread writes during the launch (`.nc`, the read-only path).
// ld_stream_u4: read once, do not allocate in L1.
// ld_gather_u4: a gathered register slice.  A hub (hub = true) is kept in L1 with evict_last; any other source does not
// allocate in L1, so the random tail of the gathers cannot evict the hubs.  The choice is a predicate on the two loads,
// not a branch, so a warp's gathers stay in flight together whatever mix of hubs its lanes hold.
__device__ __forceinline__ uint4 ld_stream_u4(const uint4* p) {
#ifndef SB200_EMU
  uint4 v;
  asm("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
#else
  return *p;
#endif
}
__device__ __forceinline__ uint4 ld_gather_u4(const uint4* p, bool hub) {
#ifndef SB200_EMU
  uint4 v = make_uint4(0, 0, 0, 0);
  asm("{\n\t.reg .pred h;\n\tsetp.ne.u32 h, %5, 0;\n\t"
      "@h ld.global.nc.L1::evict_last.v4.u32 {%0, %1, %2, %3}, [%4];\n\t"
      "@!h ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];\n\t}"
      : "+r"(v.x), "+r"(v.y), "+r"(v.z), "+r"(v.w) : "l"(p), "r"((uint32_t)hub));
  return v;
#else
  (void)hub;
  return *p;
#endif
}

}  // namespace sb200
