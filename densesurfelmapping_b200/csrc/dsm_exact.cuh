// Exactness helpers shared by the kernel files: the float-vs-double-literal compare constants, warp helpers, the
// mbarrier / bulk-copy primitives and the expression-by-expression restatement of calculate_cost
// (fusion_functions.cpp:364-387).
#pragma once
#include "dsm_device.cuh"
#include <climits>

#define MAX_ANGLE_COS 0.1     // fusion_functions.h:11

#define FULL 0xffffffffu

// ---- programmatic dependent launch (PDL) ----
// The per-frame schedule is a chain of kernels on one stream, each consuming its predecessor's output.  Every kernel
// of the chain starts with pdl_enter(): griddepcontrol.wait returns once the preceding grid has completed and its
// writes are visible (a no-op for a launch without the attribute); griddepcontrol.launch_dependents then lets the NEXT
// grid of the chain be set up -- its CTAs become resident as SM resources free up in this grid's last wave and wait at
// their own griddepcontrol.wait -- so the launch latency and the CTA ramp of the next kernel overlap this kernel's tail.
// Safe by construction: no kernel touches global memory before the wait, and a kernel is only launched with the
// attribute (pdl_launch) if it begins with pdl_enter().
#ifndef DSM_PDL
#define DSM_PDL 1
#endif
__device__ __forceinline__ void pdl_enter()
{
#if DSM_PDL
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}
template <typename... KArgs, typename... Args>
static inline void pdl_launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args &&...args)
{
#if DSM_PDL
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid, cfg.blockDim = block, cfg.dynamicSmemBytes = smem, cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at, cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kern, args...);
#else
    kern<<<grid, block, smem, s>>>(args...);
#endif
}

// Comparisons of a float against a double literal (the reference promotes the float): for a
// literal c that is not a float, with c_lo/c_hi the neighbouring floats,
//   (double)x <  c  <=>  x <  c_hi        (double)x >  c  <=>  x >  c_lo
//   (double)x >= c  <=>  x >= c_hi        (double)x <= c  <=>  x <= c_lo
// and for -c by symmetry (x > -c <=> x > -c_hi).  Used in the hot loops to keep the FP64 pipe for
// the arithmetic that really needs it; tests/test_abi.py re-derives every constant.
#define F_0p1_HI __uint_as_float(0x3dcccccdu)
#define F_0p1_LO __uint_as_float(0x3dccccccu)
#define F_0p01_HI __uint_as_float(0x3c23d70bu)
#define F_0p01_LO __uint_as_float(0x3c23d70au)
#define F_0p05_LO __uint_as_float(0x3d4cccccu)
#define F_0p2_HI __uint_as_float(0x3e4ccccdu)
#define F_0p8_HI __uint_as_float(0x3f4ccccdu)

// -------------------------------------------------------------------------------------------
// small helpers
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ int warp_excl_scan(int v, int lane, int &total)
{
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1)
    {
        int n = __shfl_up_sync(FULL, incl, o);
        if (lane >= o) incl += n;
    }
    total = __shfl_sync(FULL, incl, 31);
    return incl - v;
}

// -------------------------------------------------------------------------------------------
// mbarrier / TMA primitives (raw PTX).  One elected thread initialises a CTA's barrier, arms it with the byte count and
// issues the copies (3-D tensor boxes for the seed tiles, 1-D bulk runs for the pool records); the CTA waits for phase 0.
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); // visible to the async proxy before the first copy
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded wait: a descriptor or byte-count mistake must trap, not hang the GPU (each try_wait blocks for a hardware time slice).
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity)
{
    unsigned ok = 0;
    for (unsigned spin = 0; !ok; spin++)
    {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok)
                     : "r"(bar), "r"(parity)
                     : "memory");
        if (!ok && spin > (1u << 20)) __trap();
    }
}
__device__ __forceinline__ void tma_load_3d(unsigned dst, const CUtensorMap *map, int x, int y, int z, unsigned bar)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
                 "l"(reinterpret_cast<unsigned long long>(map)), "r"(bar), "r"(x), "r"(y), "r"(z)
                 : "memory");
}
// 1-D bulk copies: global and shared addresses 16-byte aligned, size a multiple of 16 bytes
__device__ __forceinline__ void bulk_load(unsigned dst, const void *src, unsigned bytes, unsigned bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes),
                 "r"(bar)
                 : "memory");
}
// returns once the shared-memory source has been read (it may be overwritten, or the CTA exit); the global writes complete
// asynchronously
__device__ __forceinline__ void bulk_store(void *dst, unsigned src, unsigned bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// this thread's generic-proxy shared-memory writes -> visible to the async proxy (a bulk store that follows)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// (hi, lo) split of 1.0 / (double)mean_depth for the fp32 cost filter.  mean_depth <= 0 (or NaN): the candidate has no
// depth term (:378), the pair is unused.  mean_depth < 2^-10: hi = 1e18 (its square is still finite, so a zero depth weight cannot produce a NaN) -- the depth term of such a seed exceeds 1e6 for
// every valid pixel depth (> 0.01 m, i.e. inverse < 100), so it can never be the minimum (:408, :427) and the filter
// may ignore it; if NO candidate stays below 1e6 the pixel goes to the exact path anyway.
__device__ __forceinline__ float2 split_inverse(float md)
{
    if (!(md > 0.f)) return make_float2(0.f, 0.f);
    if (md < 0.0009765625f) return make_float2(1e18f, 0.f);
    const double inv = 1.0 / (double)md;
    const float hi = (float)inv;
    return make_float2(hi, (float)(inv - (double)hi));
}

// A seed's state as the assign pass reads it: (x, y, mean_intensity, mean_depth), the fast-path and exact-path forms of
// 1 / mean_depth (only consumed when mean_depth > 0, :378) and the stable flag
__device__ __forceinline__ void store_seed(const DsmDev &d, size_t o, float x, float y, float I, float md, bool stable)
{
    d.seed[o] = make_float4(x, y, I, md);
    d.inv_md[o] = 1.0 / (double)md;
    d.seed_hl[o] = split_inverse(md);
    d.tstable[o] = stable ? DSM_STABLE : -1;
}

struct SeedC
{
    float x, y, I, md;
    double inv;
};

// Branch-free: both costs and the has-depth predicate are always computed; the caller selects.
// (When mean_depth <= 0 the hoisted 1/mean_depth is inf/NaN; the result is discarded by the select.)
__device__ __forceinline__ bool calc_cost(const SeedC &sd, float pix_i, float pix_inv, double pix_inv_d, float fx, float fy,
                                          float &nodepth, float &withdepth)
{
    const float ax = sd.x - fx, ay = sd.y - fy;
    const float dist = ax * ax + ay * ay;
    float n = dist * 0.0625f; // / (SP_SIZE/2)^2, exact power of two (:374)
    const float idf = sd.I - pix_i;
    // (double)(idf*idf) / 100.0 (:376), correctly rounded without the division subroutine:
    // q0 = RN(a*y), r = a - 100*q0 (exact in one FMA), q = RN(q0 + r*y) with y = RN(1/100) is the
    // correctly rounded quotient (Markstein); checked against x/100.0 on 3.7e8 inputs (DESIGN.md).
    const double a = (double)(idf * idf);
    const double q0 = a * 0.01;
    const double q = __fma_rn(__fma_rn(-q0, 100.0, a), 0.01, q0);
    const double nd = (double)n + q;
    n = (float)nd;
    nodepth = n;
    const bool has = sd.md > 0 && pix_inv > 0; // (:378)
    const float idd = (float)(sd.inv - pix_inv_d);                  // (:380)
    const float wd = (float)((double)n + (double)(idd * idd) * 400.0); // (:381)
    withdepth = has ? wd : n;
    return has;
}

