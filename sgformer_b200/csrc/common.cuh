// Common device helpers for the sgformer_b200 kernels (sm_90a).
// Thin inline-PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), wgmma and its shared-memory descriptors,
// cache-hinted 128-bit global loads/stores.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define SGF_OK 0
#define SGF_ERR_ARG (-1)
#define SGF_ERR_UNSUPPORTED (-2)
#define SGF_ERR_DRIVER (-3)

#define SGF_CUDA_TRY(expr)                        \
    do {                                          \
        cudaError_t _e = (expr);                  \
        if (_e != cudaSuccess) return (int)_e;    \
    } while (0)

#define SGF_LAUNCH_CHECK()                        \
    do {                                          \
        cudaError_t _e = cudaGetLastError();      \
        if (_e != cudaSuccess) return (int)_e;    \
    } while (0)

namespace sgf {

constexpr int kNumSMsDefault = 132;

__host__ inline int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
            n = kNumSMsDefault;
    }
    return n;
}

// ------------------------------------------------------------------------------------------
// small utilities
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ void unpack_bf16x2(uint32_t u, float& lo, float& hi) {
    lo = __uint_as_float(u << 16);
    hi = __uint_as_float(u & 0xffff0000u);
}

// 16-byte vector of T as 4 x u32 <-> fp32 lanes
template <typename T> struct Vec16;
template <> struct Vec16<float> {
    static constexpr int N = 4;
    __device__ __forceinline__ static void unpack(const uint4& u, float* f) {
        f[0] = __uint_as_float(u.x); f[1] = __uint_as_float(u.y);
        f[2] = __uint_as_float(u.z); f[3] = __uint_as_float(u.w);
    }
    __device__ __forceinline__ static uint4 pack(const float* f) {
        return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
    }
};
template <> struct Vec16<__nv_bfloat16> {
    static constexpr int N = 8;
    __device__ __forceinline__ static void unpack(const uint4& u, float* f) {
        unpack_bf16x2(u.x, f[0], f[1]); unpack_bf16x2(u.y, f[2], f[3]);
        unpack_bf16x2(u.z, f[4], f[5]); unpack_bf16x2(u.w, f[6], f[7]);
    }
    __device__ __forceinline__ static uint4 pack(const float* f) {
        return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
    }
};

// streaming / gather loads: read-only path, no L1 allocation (each gathered row is used once per SM)
__device__ __forceinline__ uint4 ldg_nc_na(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
// coherent variant (no .nc): for data that another GPU / copy engine writes while the kernel runs (pushed operand blocks)
__device__ __forceinline__ uint4 ldg_na(const void* p) {
    uint4 r;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
    uint32_t r;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ldg_nc_na_s32(const int* p) {
    int r;
    asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_na(void* p, const uint4& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// Bounded spin: a protocol bug traps (visible as a launch error) instead of hanging the GPU box.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) __trap();
    }
}

// ------------------------------------------------------------------------------------------
// TMA
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" :: "l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0, int32_t c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        :: "r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}

// smem tile -> global through the tensor map (rows/cols outside the tensor are clipped by the hardware)
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* smem_src, int32_t c0, int32_t c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 :: "l"(tmap), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1) : "memory");
}
// L2 prefetch of `bytes` (a multiple of 16) contiguous bytes from a 16-byte aligned global address: a hint, nothing waits on it
__device__ __forceinline__ void bulk_prefetch_l2(const void* gsrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(gsrc), "r"(bytes) : "memory");
}
// cp.async (LDGSTS): 16-byte global -> shared copies that need no destination register; a thread that reads back only what it copied
// itself needs no barrier, just wait_group.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    const uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory");
}
template <int N> __device__ __forceinline__ void bulk_wait() {
    asm volatile("cp.async.bulk.wait_group %0;" :: "n"(N) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a): D[regs] (+)= A[smem] * B[smem], bf16 x bf16 -> fp32
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory");
}
// Pins accumulator registers between an asynchronous wgmma and the wait that completes it: without it the compiler may move
// reads of the accumulators above the wait.
template <int N> __device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}

// m64 x n64 x k16.  TA / TB: 0 = K-major, 1 = MN-major operand.  scale_d = 0 overwrites D.
// Accumulator layout (thread t of the warpgroup, warp w = t / 32, lane l): d[4c + 2s + e] is row 16w + l/4 + 8s,
// column 8c + 2(l%4) + e.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

// Warp-specialised kernels of 3 warpgroups (384 threads, 168 registers each at launch): the TMA producer warpgroup gives
// registers back and the two MMA warpgroups take them (128 x 40 + 256 x 232 <= 64 K), so the accumulators stay in registers.
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(kProducerRegs)); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(kConsumerRegs)); }

// wgmma shared-memory matrix descriptor (cute::GMMA::GmmaDescriptor, sm_90):
//  [0,14) start address >> 4 | [16,30) leading byte offset >> 4 | [32,46) stride byte offset >> 4 |
//  [49,52) base offset = 0 (tiles are 1024-byte aligned) | [62,64) layout type (1 = SWIZZLE_128B).
// K-major SW128 (rows of 64 bf16 = 128 bytes): SBO = 1024 (8-row groups), LBO unused; the k-th 16-element step starts 32k
// bytes further.  MN-major SW128: LBO = stride between 64-element MN chunks, SBO = stride between 8-row K groups.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}

// ------------------------------------------------------------------------------------------
// counter-based dropout RNG (no mask tensor: the backward recomputes the mask)
// ------------------------------------------------------------------------------------------
// Dropout of one 16-byte chunk (VN = 4 or 8 elements): one 64-bit hash per 4 elements, 16 random bits per element.
// thr16 = round(p * 65536); an element is kept when its 16 bits >= thr16 and scaled by inv_keep = 65536 / (65536 - thr16).
// The mask is a pure function of (seed, chunk_id) so the backward recomputes it (chunk_id = row * chunks_per_row + chunk).
template <int VN>
__device__ __forceinline__ void dropout_chunk(uint64_t seed, uint64_t chunk_id, uint32_t thr16, float inv_keep, float* f) {
#pragma unroll
    for (int k = 0; k < VN / 4; ++k) {
        uint64_t x = seed + (chunk_id * (VN / 4) + k) * 0x9E3779B97F4A7C15ULL;
        x ^= x >> 33; x *= 0xff51afd7ed558ccdULL;
        x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL;
        x ^= x >> 33;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t u = static_cast<uint32_t>(x >> (16 * j)) & 0xFFFFu;
            f[4 * k + j] *= (u >= thr16) ? inv_keep : 0.f;
        }
    }
}
// The device epoch word registered by sgf_set_dropout_epoch (rowops.cu), or null.
const uint64_t* dropout_epoch_word();

// Activation codes of the BatchNorm kernels' `use_relu` argument: 0 none, 1 ReLU, kActElu ELU (alpha 1; GAT's F.elu).
constexpr int kActElu = 2;

__host__ __device__ __forceinline__ uint32_t dropout_thr16(float p) { return static_cast<uint32_t>(p * 65536.f + 0.5f); }
__host__ __device__ __forceinline__ float dropout_inv_keep(uint32_t thr16) { return 65536.f / (65536.f - static_cast<float>(thr16)); }

}  // namespace sgf
