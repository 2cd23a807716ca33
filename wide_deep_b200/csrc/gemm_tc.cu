// wgmma (Hopper warp-group tensor core) engine for the MLP GEMMs on sm_90a.
//
//   C[M,N] = sum_k A[M,k] * B[N,k]     fp32 operands, both K-contiguous ("TN"), fp32 accumulate in registers
//
// fp32-faithful products on the tf32 pipe (3xTF32): every operand tile is split in shared memory into
//   hi = x with the low 13 mantissa bits cleared (exactly representable in tf32)     lo = x - hi (exact)
// and three MMAs accumulate  a_lo*b_hi + a_hi*b_lo + a_hi*b_hi  into the same accumulator; the dropped
// a_lo*b_lo term is below 2^-22 relative, i.e. at fp32 rounding level, which is what the 1e-4 logit parity bar
// (BASELINE.json) needs and what a single tf32 pass (2^-11) cannot give.
//
// One persistent CTA per SM loops over 128 x 128 output tiles, K loop over 32-float = 128-byte blocks.  Four warp groups:
//   group 0     TMA producer (one elected thread): cp.async.bulk.tensor.2d of the raw fp32 A / B blocks (128B-swizzled)
//               into the "hi" buffers of a stage ring, completion on mbarrier full[s]
//   group 1     splitters: wait full[s], rewrite the block in place as hi and write lo beside it (element-wise,
//               so the swizzle never has to be decoded), fence.proxy.async, arrive split[s]
//   groups 2-3  consumers, 64 tile rows each: wait split[s], 4 k-steps x 3 wgmma.mma_async m64n128k8 tf32, release the stage
//               on empty[s] once that batch has retired; then the epilogue straight from the accumulator fragment: fused
//               bias + activation + BN-affine (+ transposed copy) or plain / accumulating / split-K store
// The producer and the splitters hand registers to the consumers (setmaxnreg) and run ahead into the next tile while the
// consumers store the current one.  Inputs that run past M, N or K are zero-filled by TMA (tensor maps carry the true
// extents).
#include <cuda.h>
#include <stdlib.h>

#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "gemm.cuh"
#include "wgmma_ptx.cuh"

namespace wd {

constexpr int TBM = 128;        // tile rows: two consumer warp groups x wgmma M = 64
constexpr int TBN = 128;        // tile columns: 64 accumulator registers per consumer thread is what four warp groups leave room for
constexpr int TBK = 32;         // floats per k-block = one 128-byte swizzle row
constexpr int TSTAGES = 3;
constexpr int TC_THREADS = 512;

struct TcMaps {
    CUtensorMap a[kMaxSegs];
    CUtensorMap b;
    CUtensorMap b_lo;          // pre-split weights: b = hi copy, b_lo = lo copy
};

// ---------------------------------------------------------------------------------------------- kernel
// SPLIT3: three products (3xTF32), else one (tc1x).  The forward and data-gradient GEMMs of 3xTF32 (BPRE) read the weights
// already split into hi / lo copies (two tensor maps) and split only A here.
template <int MODE, bool SPLIT3>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_gemm_kernel(const __grid_constant__ TcMaps maps, int nseg, int4 segk01, int4 segk23,
                                                               int M, int N, int ktot, int ksplit_len, int nsplit, Epi ep) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr bool BPRE = SPLIT3 && MODE != EPI_WGRAD;
    constexpr int A_BYTES = TBM * 128, B_BYTES = TBN * 128;
    constexpr int STAGE_BYTES = (SPLIT3 ? 2 : 1) * (A_BYTES + B_BYTES);
    constexpr int NST = TSTAGES;
    auto a_hi = [&](int s) { return base + s * STAGE_BYTES; };
    auto b_hi = [&](int s) { return base + s * STAGE_BYTES + A_BYTES; };
    auto a_lo = [&](int s) { return base + s * STAGE_BYTES + A_BYTES + B_BYTES; };
    auto b_lo = [&](int s) { return base + s * STAGE_BYTES + 2 * A_BYTES + B_BYTES; };
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + NST * STAGE_BYTES);
    uint64_t* full = bars; uint64_t* split = bars + NST; uint64_t* empty = bars + 2 * NST;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    const int tiles_n = (N + TBN - 1) / TBN, tiles_m = (M + TBM - 1) / TBM;
    const int ntiles = tiles_n * tiles_m * nsplit;
    auto tile_range = [&](int tile, int& m0, int& n0, int& z, int& kbeg, int& nkb) {
        z = tile / (tiles_n * tiles_m);
        int r = tile % (tiles_n * tiles_m);
        m0 = (r / tiles_n) * TBM;
        n0 = (r % tiles_n) * TBN;
        kbeg = 0;
        int kend = ktot;
        if (MODE == EPI_WGRAD) { kbeg = z * ksplit_len; kend = min(ktot, kbeg + ksplit_len); }
        nkb = kend > kbeg ? (kend - kbeg + TBK - 1) / TBK : 0;
    };

    if (threadIdx.x == 0) {
        for (int s = 0; s < NST; ++s) { mbar_init(&full[s], 1); mbar_init(&split[s], 128); mbar_init(&empty[s], 8); }   // empty: one arrival per consumer warp
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------------ TMA producer
        reg_dealloc<40>();
        if (warp == 0 && lane == 0) {
            const int segk[kMaxSegs] = {segk01.x, segk01.y, segk01.z, segk01.w, segk23.x, segk23.y, segk23.z, segk23.w};
            int g = 0;
            for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
                int m0, n0, z, kbeg, nkb;
                tile_range(tile, m0, n0, z, kbeg, nkb);
                for (int kb = 0; kb < nkb; ++kb, ++g) {
                    const int s = g % NST, it = g / NST;
                    if (it > 0) mbar_wait(&empty[s], (it - 1) & 1);
                    int kg = kbeg + kb * TBK;
                    int seg = 0, kk = kg;
                    while (seg < nseg - 1 && kk >= segk[seg]) { kk -= segk[seg]; ++seg; }
                    mbar_expect_tx(&full[s], A_BYTES + (BPRE ? 2 : 1) * B_BYTES);
                    tma_load_2d(a_hi(s), &maps.a[seg], &full[s], kk, m0);
                    tma_load_2d(b_hi(s), &maps.b, &full[s], kg, n0);
                    if (BPRE) tma_load_2d(b_lo(s), &maps.b_lo, &full[s], kg, n0);
                }
            }
        }
    } else if (wg == 1) {
        // ------------------------------------------------------------------ splitters
        reg_dealloc<72>();
        if (SPLIT3) {
            const int t = threadIdx.x - 128;                    // 0..127
            int g = 0;
            for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
                int m0, n0, z, kbeg, nkb;
                tile_range(tile, m0, n0, z, kbeg, nkb);
                for (int kb = 0; kb < nkb; ++kb, ++g) {
                    const int s = g % NST, it = g / NST;
                    mbar_wait(&full[s], it & 1);
                    float4* ah = reinterpret_cast<float4*>(a_hi(s)); float4* al = reinterpret_cast<float4*>(a_lo(s));
                    float4* bh = reinterpret_cast<float4*>(b_hi(s)); float4* bl = reinterpret_cast<float4*>(b_lo(s));
                    auto split4 = [](float4 x, float4& hi, float4& lo) {
                        hi.x = __uint_as_float(__float_as_uint(x.x) & 0xFFFFE000u); lo.x = x.x - hi.x;
                        hi.y = __uint_as_float(__float_as_uint(x.y) & 0xFFFFE000u); lo.y = x.y - hi.y;
                        hi.z = __uint_as_float(__float_as_uint(x.z) & 0xFFFFE000u); lo.z = x.z - hi.z;
                        hi.w = __uint_as_float(__float_as_uint(x.w) & 0xFFFFE000u); lo.w = x.w - hi.w;
                    };
#pragma unroll
                    for (int i = 0; i < A_BYTES / 16 / 128; ++i) {
                        float4 x = ah[t + i * 128], hi, lo;
                        split4(x, hi, lo);
                        ah[t + i * 128] = hi; al[t + i * 128] = lo;
                    }
                    if (!BPRE) {
#pragma unroll
                        for (int i = 0; i < B_BYTES / 16 / 128; ++i) {
                            float4 x = bh[t + i * 128], hi, lo;
                            split4(x, hi, lo);
                            bh[t + i * 128] = hi; bl[t + i * 128] = lo;
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
                    mbar_arrive(&split[s]);
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ consumers: warp group cw owns rows [64 cw, 64 cw + 64)
        reg_alloc<200>();
        const int cw = wg - 2;
        float d[TBN / 2];
        int g = 0;
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            int m0, n0, z, kbeg, nkb;
            tile_range(tile, m0, n0, z, kbeg, nkb);
            if (nkb == 0) {
#pragma unroll
                for (int i = 0; i < TBN / 2; ++i) d[i] = 0.f;
            }
            int prev = -1;
            for (int kb = 0; kb < nkb; ++kb, ++g) {
                const int s = g % NST, it = g / NST;
                mbar_wait(SPLIT3 ? &split[s] : &full[s], it & 1);
                const uint32_t sa_hi = smem_u32(a_hi(s)) + cw * 8192, sa_lo = smem_u32(a_lo(s)) + cw * 8192;   // 64 rows x 128 B per group
                const uint32_t sb_hi = smem_u32(b_hi(s)), sb_lo = smem_u32(b_lo(s));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < TBK / 8; ++k) {
                    const uint32_t off = k * 32;          // 8 tf32 = 32 bytes inside the 128-byte swizzle row
                    const uint32_t acc = (kb > 0 || k > 0) ? 1u : 0u;
                    if (SPLIT3) {
                        wgmma_tf32(d, make_desc(sa_lo + off), make_desc(sb_hi + off), acc);
                        wgmma_tf32(d, make_desc(sa_hi + off), make_desc(sb_lo + off), 1u);
                        wgmma_tf32(d, make_desc(sa_hi + off), make_desc(sb_hi + off), 1u);
                    } else {
                        wgmma_tf32(d, make_desc(sa_hi + off), make_desc(sb_hi + off), acc);
                    }
                }
                wgmma_commit();
                if (prev >= 0) {
                    wgmma_wait<1>();                              // the batch that read stage `prev` has retired
                    if (lane == 0) mbar_arrive(&empty[prev]);
                }
                prev = s;
            }
            wgmma_wait<0>();                                      // the accumulator is final
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

            // ---- epilogue from the accumulator fragment: rows r0 and r0 + 8, columns n0 + 8 j + 2 (lane % 4) + {0, 1}
            const int r0 = m0 + cw * 64 + (warp & 3) * 16 + (lane >> 2);
            const int cq = 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < TBN / 8; ++j) {
                const int c = n0 + 8 * j + cq;
                if (n0 + 8 * j >= N) continue;
                if (MODE == EPI_FWD) {
                    const bool in0 = c < ep.n_logical, in1 = c + 1 < ep.n_logical;
                    const float b0 = in0 ? __ldg(ep.bias + c) : 0.f, b1 = in1 ? __ldg(ep.bias + c + 1) : 0.f;
                    const float g0 = (in0 && ep.bn) ? __ldg(ep.gamma + c) * 0.99950037468777f : 1.f;
                    const float g1 = (in1 && ep.bn) ? __ldg(ep.gamma + c + 1) * 0.99950037468777f : 1.f;
                    const float e0 = (in0 && ep.bn) ? __ldg(ep.beta + c) : 0.f, e1 = (in1 && ep.bn) ? __ldg(ep.beta + c + 1) : 0.f;
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int r = r0 + 8 * hh;
                        const bool rv = r < ep.m_valid;              // rows >= m_valid are written as zero (transposed padding)
                        float a0 = 0.f, a1 = 0.f, h0 = 0.f, h1 = 0.f;
                        if (rv && in0) { a0 = ep.act == WD_ACT_RELU ? fmaxf(d[4 * j + 2 * hh] + b0, 0.f) : act_fwd(ep.act, d[4 * j + 2 * hh] + b0); h0 = fmaf(a0, g0, e0); }
                        if (rv && in1) { a1 = ep.act == WD_ACT_RELU ? fmaxf(d[4 * j + 2 * hh + 1] + b1, 0.f) : act_fwd(ep.act, d[4 * j + 2 * hh + 1] + b1); h1 = fmaf(a1, g1, e1); }
                        if (r < M) {
                            const int64_t o = (int64_t)r * ep.ldh + c;
                            if (ep.A_out != ep.H_out) *reinterpret_cast<float2*>(ep.A_out + o) = make_float2(a0, a1);
                            *reinterpret_cast<float2*>(ep.H_out + o) = make_float2(h0, h1);
                        }
                        if (ep.HT) {                                 // 8 lanes = 8 consecutive m: whole 32-byte sectors
                            ep.HT[(int64_t)c * ep.ldt + r] = h0;
                            ep.HT[(int64_t)(c + 1) * ep.ldt + r] = h1;
                        }
                    }
                } else {
                    float* Cb = ep.C + (MODE == EPI_WGRAD ? (int64_t)z * ep.split_stride : 0);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int r = r0 + 8 * hh;
                        if (r >= M) continue;
                        float2* pc = reinterpret_cast<float2*>(Cb + (int64_t)r * ep.ldc + c);
                        float2 o = make_float2(d[4 * j + 2 * hh], d[4 * j + 2 * hh + 1]);
                        if (MODE == EPI_STORE && ep.accumulate) { const float2 p = *pc; o.x += p.x; o.y += p.y; }
                        *pc = o;
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- host
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeFn g_encode = nullptr;

static int get_encode() {
    if (g_encode) return WD_OK;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || !fn) { set_error("cuTensorMapEncodeTiled unavailable: %s", cudaGetErrorString(e)); return WD_ECUDA; }
    g_encode = (EncodeFn)fn;
    return WD_OK;
}

// Encoded tensor maps are cached by (base, shape, pitch, box, element size): a train step re-creates the same ~100 maps every
// time, and cuTensorMapEncodeTiled costs about a microsecond each on the launching thread — which matters wherever steps are
// launched eagerly (data-parallel steps, profiling), not replayed from a CUDA graph.
struct MapKey {
    const void* p; int rows, cols, ld, box_rows, esize;
    bool operator==(const MapKey& o) const { return p == o.p && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows && esize == o.esize; }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        uint64_t h = (uint64_t)(uintptr_t)k.p * 0x9E3779B97F4A7C15ull;
        h ^= ((uint64_t)(uint32_t)k.rows << 32 | (uint32_t)k.cols) * 0xC2B2AE3D27D4EB4Full;
        h ^= ((uint64_t)(uint32_t)k.ld << 20 | (uint64_t)(uint32_t)k.box_rows << 4 | (uint32_t)k.esize) * 0x165667B19E3779F9ull;
        return (size_t)(h ^ (h >> 29));
    }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;
static std::mutex g_map_mutex;
static bool map_cache_get(const MapKey& k, CUtensorMap* out) {
    std::lock_guard<std::mutex> lock(g_map_mutex);
    auto it = g_map_cache.find(k);
    if (it == g_map_cache.end()) return false;
    *out = it->second;
    return true;
}
static void map_cache_put(const MapKey& k, const CUtensorMap& v) {
    std::lock_guard<std::mutex> lock(g_map_mutex);
    if (g_map_cache.size() > 4096) g_map_cache.clear();          // models come and go (tests): keep the table bounded
    g_map_cache[k] = v;
}
// a freed model's buffers may be handed out again with another shape: drop every cached map when a model dies
void tc_map_cache_clear() {
    std::lock_guard<std::mutex> lock(g_map_mutex);
    g_map_cache.clear();
}

int make_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, const void* ptr, int rows, int cols, int ld, int box_rows) {
    int rc = get_encode();
    if (rc) return rc;
    const int esize = dtype == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? 4 : 2;       // fp32 or bf16
    const MapKey key{ptr, rows, cols, ld, box_rows, esize};
    if (map_cache_get(key, map)) return WD_OK;
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
    cuuint32_t box[2] = {(cuuint32_t)(128 / esize), (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(map, dtype, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d) rows=%d cols=%d ld=%d element=%d bytes", (int)r, rows, cols, ld, esize);
        return WD_ECUDA;
    }
    map_cache_put(key, *map);
    return WD_OK;
}

template <int MODE, bool SPLIT3>
static int launch_tc(WdModel* m, const TcMaps& maps, int nseg, const int* segk, int M, int N, int ktot, int splits, int ksplit_len, const Epi& ep) {
    constexpr int A_BYTES = TBM * 128, B_BYTES = TBN * 128;
    constexpr int NST = TSTAGES;
    constexpr int smem = NST * (SPLIT3 ? 2 : 1) * (A_BYTES + B_BYTES) + 1024 + 128;
    int4 s01 = make_int4(segk[0], segk[1], segk[2], segk[3]), s23 = make_int4(segk[4], segk[5], segk[6], segk[7]);
    static bool configured = false;
    static int num_sms = 0;
    if (!configured) {
        WD_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<MODE, SPLIT3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        WD_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, m->device));
        configured = true;
    }
    const int nsplit = MODE == EPI_WGRAD ? splits : 1;
    const int ntiles = ((N + TBN - 1) / TBN) * ((M + TBM - 1) / TBM) * nsplit;
    tc_gemm_kernel<MODE, SPLIT3><<<ntiles < num_sms ? ntiles : num_sms, TC_THREADS, smem, m->stream>>>(maps, nseg, s01, s23, M, N, ktot, ksplit_len, nsplit, ep);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

int tc_gemm(WdModel* m, int mode, const GemmA& A, const GemmB& B, int M, int N, const Epi& ep, int splits, int ksplit_len) {
    constexpr CUtensorMapDataType F32 = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    int rc;
    if (N % 32 != 0 || A.n > kMaxSegs) return WD_EUNSUPPORTED;
    TcMaps maps;
    int segk[kMaxSegs] = {0};
    int ktot = 0;
    for (int s = 0; s < A.n; ++s) {
        if (A.k[s] % TBK != 0 && A.n > 1) return WD_EUNSUPPORTED;     // interior segment boundaries must sit on k-block edges
        if ((rc = make_tensor_map(&maps.a[s], F32, A.ptr[s], M, A.k[s], A.ld[s], TBM))) return rc;
        segk[s] = A.k[s];
        ktot += A.k[s];
    }
    for (int s = A.n; s < kMaxSegs; ++s) maps.a[s] = maps.a[0];
    const bool split3 = m->gemm_engine == WD_GEMM_TC3X;
    const bool bpre = split3 && mode != EPI_WGRAD;                     // (tc_gemm_kernel's BPRE)
    if (bpre && (!B.tf32_hi || !B.tf32_lo)) { set_error("3xTF32 GEMM engine: weights without hi/lo copies"); return WD_EINVAL; }
    if ((rc = make_tensor_map(&maps.b, F32, bpre ? B.tf32_hi : B.ptr, N, ktot, B.ld, TBN))) return rc;
    if (bpre) { if ((rc = make_tensor_map(&maps.b_lo, F32, B.tf32_lo, N, ktot, B.ld, TBN))) return rc; }
    else maps.b_lo = maps.b;
    if (mode == EPI_WGRAD) ksplit_len = (ksplit_len + TBK - 1) / TBK * TBK;
#define WD_TC_LAUNCH(MODE_)                                                                                      \
    return split3 ? launch_tc<MODE_, true>(m, maps, A.n, segk, M, N, ktot, splits, ksplit_len, ep)              \
                  : launch_tc<MODE_, false>(m, maps, A.n, segk, M, N, ktot, splits, ksplit_len, ep)
    if (mode == EPI_FWD) WD_TC_LAUNCH(EPI_FWD);
    if (mode == EPI_STORE) WD_TC_LAUNCH(EPI_STORE);
    WD_TC_LAUNCH(EPI_WGRAD);
#undef WD_TC_LAUNCH
}

}  // namespace wd
