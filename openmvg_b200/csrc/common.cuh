// common.cuh — error plumbing, owning buffers, checked launches, the device check and the sm_90a PTX wrappers (mbarrier,
// TMA, wgmma) shared by match.cu, geom.cu and ba.cu.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <string>
#include <map>
#include <mutex>
#include <unordered_map>
#include <utility>

#include "../../include/omvg_b200.h"

namespace omvg {

inline std::string &last_error() { static thread_local std::string e; return e; }
inline int fail(int code, const char *fmt, ...) {
  char buf[512]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  last_error() = buf; return code;
}
#define OMVG_CUDA(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
  return ::omvg::fail(OMVG_E_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } while (0)

// ----------------------------------------------------------------------------- caching device allocator
// Adjust()/Match() are called many times by the SfM engines (BA / outlier-rejection / BA loops): cudaMalloc and
// cudaFree of ~100 work buffers cost more than a whole solve, so released buffers are kept per device and
// handed out again (best fit within 25 % slack).  omvg_trim_cache() returns everything to the driver.
struct DevPool {
  std::mutex mu;
  std::multimap<size_t, void *> free_[16];
  std::unordered_map<void *, std::pair<size_t, int>> live;
  size_t cached = 0;
};
inline DevPool &dev_pool() { static DevPool p; return p; }
inline cudaError_t pool_malloc(void **out, size_t bytes) {
  int dev = 0; cudaGetDevice(&dev); dev &= 15;
  bytes = (bytes + 511) & ~size_t(511);
  DevPool &P = dev_pool();
  { std::lock_guard<std::mutex> g(P.mu);
    auto it = P.free_[dev].lower_bound(bytes);
    if (it != P.free_[dev].end() && it->first <= bytes + bytes / 4 + 4096) {
      *out = it->second; P.live[*out] = {it->first, dev}; P.cached -= it->first; P.free_[dev].erase(it); return cudaSuccess; } }
  cudaError_t e = cudaMalloc(out, bytes);
  if (e != cudaSuccess) {                                   // out of memory: drop the cache and retry once
    { std::lock_guard<std::mutex> g(P.mu); for (auto &kv : P.free_[dev]) cudaFree(kv.second); for (auto &kv : P.free_[dev]) P.cached -= kv.first; P.free_[dev].clear(); }
    cudaGetLastError(); e = cudaMalloc(out, bytes);
  }
  if (e == cudaSuccess) { std::lock_guard<std::mutex> g(P.mu); P.live[*out] = {bytes, dev}; }
  return e;
}
inline void pool_free(void *p) {
  if (!p) return;
  DevPool &P = dev_pool();
  std::lock_guard<std::mutex> g(P.mu);
  auto it = P.live.find(p);
  if (it == P.live.end()) { cudaFree(p); return; }
  const size_t bytes = it->second.first; const int dev = it->second.second; P.live.erase(it);
  if (P.cached + bytes > (size_t(16) << 30)) { cudaFree(p); return; }
  P.free_[dev].emplace(bytes, p); P.cached += bytes;
}
inline void pool_trim() {
  DevPool &P = dev_pool();
  std::lock_guard<std::mutex> g(P.mu);
  for (int d = 0; d < 16; ++d) { for (auto &kv : P.free_[d]) cudaFree(kv.second); P.free_[d].clear(); }
  P.cached = 0;
}

// ----------------------------------------------------------------------------- owning buffers
// Where a buffer's memory comes from: the caching pool above, the driver (cudaFree hands the memory back at once), or
// pinned host memory.
struct PoolAlloc { static cudaError_t get(void **p, size_t b) { return pool_malloc(p, b); } static void put(void *p) { pool_free(p); } };
struct CudaAlloc { static cudaError_t get(void **p, size_t b) { return cudaMalloc(p, b); } static void put(void *p) { cudaFree(p); } };
struct PinnedAlloc { static cudaError_t get(void **p, size_t b) { return cudaMallocHost(p, b); } static void put(void *p) { cudaFreeHost(p); } };

// n elements of T, released when the buffer is destroyed or overwritten; movable, not copyable
template <typename T, typename A = PoolAlloc> struct DevBuf {
  T *p = nullptr; size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  DevBuf &operator=(DevBuf &&o) noexcept { if (this != &o) { release(); std::swap(p, o.p); std::swap(n, o.n); } return *this; }
  ~DevBuf() { release(); }
  int alloc(size_t count) { release(); if (!count) return OMVG_OK; OMVG_CUDA(A::get(reinterpret_cast<void **>(&p), count * sizeof(T))); n = count; return OMVG_OK; }
  int reserve(size_t count) { return count <= n ? OMVG_OK : alloc(count); }   // grow only; the old contents are lost
  void release() { if (p) A::put(p); p = nullptr; n = 0; }
};

// ----------------------------------------------------------------------------- launches
// Every kernel of a context (anything with a stream and a launch counter) is launched through launch() or launch_coop()
// (grid-wide barriers), which check the launch and count it.
template <typename C, typename... P, typename... A>
int launch(C *c, void (*k)(P...), dim3 grid, dim3 block, size_t smem, A &&...args) {
  k<<<grid, block, smem, c->stream>>>(std::forward<A>(args)...);
  OMVG_CUDA(cudaGetLastError());
  ++c->launches; return OMVG_OK;
}
template <typename T> struct NoDeduce { using type = T; };
template <typename C, typename... P>
int launch_coop(C *c, void (*k)(P...), dim3 grid, dim3 block, size_t smem, typename NoDeduce<P>::type... args) {
  void *argv[] = {&args...};
  OMVG_CUDA(cudaLaunchCooperativeKernel((void *)k, grid, block, argv, smem, c->stream));
  ++c->launches; return OMVG_OK;
}

// the CUDA device exists and is an sm_90 part; its SM count out (attributes: cudaGetDeviceProperties costs milliseconds)
inline int check_device(int device, int *n_sms) {
  int n = 0; OMVG_CUDA(cudaGetDeviceCount(&n));
  if (device < 0 || device >= n) return fail(OMVG_E_CUDA, "no CUDA device %d (found %d)", device, n);
  int cc_major = 0, cc_minor = 0;
  OMVG_CUDA(cudaDeviceGetAttribute(&cc_major, cudaDevAttrComputeCapabilityMajor, device));
  OMVG_CUDA(cudaDeviceGetAttribute(&cc_minor, cudaDevAttrComputeCapabilityMinor, device));
  OMVG_CUDA(cudaDeviceGetAttribute(n_sms, cudaDevAttrMultiProcessorCount, device));
  if (cc_major != 9 || cc_minor != 0) return fail(OMVG_E_CUDA, "device %d is sm_%d%d; this library is sm_90a only", device, cc_major, cc_minor);
  return OMVG_OK;
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("{ .reg .b64 t; mbarrier.arrive.shared::cta.b64 t, [%0]; }" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("{ .reg .b64 t; mbarrier.arrive.expect_tx.shared::cta.b64 t, [%0], %1; }" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must trap, not hang the GPU.  (No printf here: a function call inside the wgmma
// kernel makes ptxas serialise its MMAs.)
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) { if (++spins > (1u << 26)) __trap(); }
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const void *tmap, int x, int y, uint64_t *bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               :: "r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void bulk_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const void *tmap) { asm volatile("prefetch.tensormap [%0];" :: "l"(tmap) : "memory"); }

// ----------------------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor of a K-major operand tile (sm_90 layout): start address, leading / stride byte
// offsets, swizzle mode in bits 62-63 (1 = 128-byte, 3 = 32-byte).  Rows of 128 bytes under the 128-byte swizzle
// (what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B) form 8-row x 128-B atoms 1024 B apart; a K-slice of 32 bytes
// inside the row is addressed by advancing the start address.  Rows of 32 bytes under the 32-byte swizzle form
// 8-row x 32-B atoms 256 B apart.  The leading byte offset is unused for swizzled K-major tiles.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t sbo, uint32_t layout) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);        // start address  [0,14)
  d |= (uint64_t)1 << 16;                              // LBO            [16,30)
  d |= (uint64_t)(sbo >> 4) << 32;                     // SBO            [32,46)
  d |= (uint64_t)layout << 62;                         // swizzle mode   [62,64)
  return d;
}
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) { return gmma_desc(smem_addr, 1024, 1); }
__device__ __forceinline__ uint64_t make_kmajor_sw32_desc(uint32_t smem_addr) { return gmma_desc(smem_addr, 256, 3); }

#define OMVG_ACC128(d) \
  "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), \
  "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), \
  "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), \
  "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), \
  "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), \
  "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), \
  "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), \
  "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), \
  "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), \
  "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), \
  "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), \
  "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), \
  "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), \
  "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]), \
  "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]), \
  "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])

// D[64 x 256] (+)= A[smem desc, 64 x 32] * B[smem desc, 256 x 32]^T, u8 x u8 (or u8 x s8) -> s32, one warpgroup.
// Thread t of the warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) and columns 8 j + 2 (t % 4) (+ 1):
// d[4 j + 0..1] = row r, d[4 j + 2..3] = row r + 8.
#define OMVG_WGMMA_ASM(BTYPE) \
  "{ .reg .pred p; setp.ne.b32 p, %130, 0; wgmma.mma_async.sync.aligned.m64n256k32.s32.u8." BTYPE " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p; }"
template <bool SIGNED_B>
__device__ __forceinline__ void wgmma_m64n256k32(int32_t (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (SIGNED_B)
    asm volatile(OMVG_WGMMA_ASM("s8") : OMVG_ACC128(d) : "l"(adesc), "l"(bdesc), "r"(accumulate) : "memory");
  else
    asm volatile(OMVG_WGMMA_ASM("u8") : OMVG_ACC128(d) : "l"(adesc), "l"(bdesc), "r"(accumulate) : "memory");
}
// wgmma.fence before the first MMA of a tile: orders the earlier register reads of the accumulators (the epilogue)
// before the MMAs overwrite them.
__device__ __forceinline__ void wgmma_fence(int32_t (&d)[128]) { asm volatile("wgmma.fence.sync.aligned;" : OMVG_ACC128(d) :: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait for every committed group, with the accumulators as in/out operands so that no use of them can be scheduled
// above the wait
__device__ __forceinline__ void wgmma_wait_all(int32_t (&d)[128]) { asm volatile("wgmma.wait_group.sync.aligned 0;" : OMVG_ACC128(d) :: "memory"); }

}  // namespace omvg
