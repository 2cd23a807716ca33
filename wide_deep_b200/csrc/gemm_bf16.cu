// 3xBF16 wgmma engine for the MLP GEMMs on sm_90a (the engine bench.py runs).
//
//   C[M,N] = sum_k A[M,k] * B[N,k]      fp32 values, fp32 accumulation in registers
//
// Every fp32 operand exists in HBM as two bf16 copies, hi = bf16_rn(x) and lo = bf16_rn(x - hi), written by the kernel that
// PRODUCED the operand (forward epilogue, x0_split_kernel, act_bn_bwd_q_kernel, logits_act_bwd_q_kernel, dense_vec_kernel), so
// this kernel moves and multiplies bf16 only: per 64-element k-block four TMA tiles (A_hi, A_lo, B_hi, B_lo; 128-byte swizzle) and
// 4 k-steps x 3 wgmma.mma_async (a_lo*b_hi + a_hi*b_lo + a_hi*b_hi) into one fp32 accumulator.  hi + lo represents x to
// 2^-17 and the dropped a_lo*b_lo term is below 2^-16, so one product carries ~1e-5 relative error (random signs, so a long dot
// product does better).  That is a FAST mode: it is held to the 1e-4 logit bar on the benchmarked configuration (bench.py
// re-checks it against the oracle in the same run, tests/test_gpu_bench_engine.py under pytest) but is not fp32-faithful the way
// the 3xTF32 engine (gemm_tc.cu, 2^-21) is; it moves half the shared-memory bytes per flop and needs no in-kernel splitting pass.
//
// Operand majors.  Forward: A = activations [m][k] (K-major), B = weights W[k][n] (MN-major: n contiguous) — no transposed weight
// copy exists.  Data gradient: A = dZ [m][n] and B = W[k_in][n], both K-major over n.  Weight gradient: A = layer input [b][k_in]
// and B = dZ [b][n], both MN-major with the batch as the reduction dimension — no transposed activation copies exist either,
// and TMA zero-fills the batch tail.  An MN-major operand is fetched as 64-column boxes (64 k-rows x 128 B, 128-byte swizzle);
// its descriptor uses LBO = one box (8 KB) between 64-wide column groups and SBO = 1 KB between 8-row k groups.
//
// One persistent CTA per SM, three warp groups: group 0 = TMA producer (one elected thread, registers handed over with
// setmaxnreg), groups 1-2 = consumers, each owning 64 rows of the 128 x 128 tile in registers (64 accumulators per thread).
// A consumer releases a pipeline stage once the wgmma batch that read it has retired (wait_group 1: the next batch is already
// queued), and the producer runs ahead into the next tile while the consumers store the current one.  Forward epilogue = bias +
// activation + BN-affine straight from the accumulator fragment; it stores the post-activation values (fp32, for the backward),
// the layer output as bf16 hi/lo copies (what the next layer and the weight gradient read) and, only for layers the logits layer
// reads, the fp32 layer output.  A quad of lanes owns 8 consecutive columns of a row, so every fp32 store instruction writes
// whole 32-byte sectors; the bf16 copies of two column groups are exchanged within the quad and stored together, so they
// write whole sectors too (with half-sector stores the forward launches took ~20 % longer).
// The forward epilogue's per-column constants (bias, gamma' and beta of the tile's 128 columns) are fetched before the main loop
// and handed to the epilogue through 3 KB of shared memory, so no global-load latency sits between its stores.
#include <cuda.h>
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "gemm.cuh"
#include "wgmma_ptx.cuh"

namespace wd {

namespace {

constexpr int QBM = 128;         // tile rows: two warp groups x wgmma M = 64
constexpr int QBN = 128;         // tile columns (wgmma N)
constexpr int QNST = 3;          // pipeline stages of 64 KB: 192 KB of the 227 KB a block may use
constexpr int QBK = 64;          // bf16 elements per k-block = one 128-byte swizzle row
constexpr int Q_THREADS = 384;   // warp group 0 TMA, warp groups 1-2 MMA + epilogue

struct QMaps {
    CUtensorMap a_hi[kMaxSegs], a_lo[kMaxSegs];
    CUtensorMap b_hi, b_lo;
};
struct QSegs { int n; int k[kMaxSegs]; int koff[kMaxSegs]; };

// optional timeline probe of CTA 0 (WD_GEMM_PROBE=1): globaltimer stamps per launch slot, read back by wd_debug_gemm_probe.
// 0 kernel start, 1 first operands landed, 2 / 3 main loop of the first / last tile done, 4 / 5 epilogue of the first / last tile done
__device__ unsigned long long g_probe[32 * 8];
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define PROBE(i) do { if (probe >= 0 && blockIdx.x == 0 && (threadIdx.x & 127) == 0) g_probe[probe * 8 + (i)] = gtime(); } while (0)

template <int MODE>
__global__ void __launch_bounds__(Q_THREADS, 1) tc_gemm_bf16_kernel(const __grid_constant__ QMaps maps, const QSegs segs, int M, int N, int ktot,
                                                                   int ksplit_len, int nsplit, Epi ep, int probe) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr bool A_MN = MODE == EPI_WGRAD;                       // operand stored with its M / N index contiguous
    constexpr bool B_MN = MODE == EPI_FWD || MODE == EPI_WGRAD;
    constexpr int A_BYTES = QBM * 128, B_BYTES = QBN * 128;
    constexpr int STAGE_BYTES = 2 * (A_BYTES + B_BYTES);
    auto a_hi = [&](int s) { return base + s * STAGE_BYTES; };
    auto a_lo = [&](int s) { return base + s * STAGE_BYTES + A_BYTES; };
    auto b_hi = [&](int s) { return base + s * STAGE_BYTES + 2 * A_BYTES; };
    auto b_lo = [&](int s) { return base + s * STAGE_BYTES + 2 * A_BYTES + B_BYTES; };
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + QNST * STAGE_BYTES);
    uint64_t* full = bars; uint64_t* empty = bars + QNST;
    float* epi_vec = reinterpret_cast<float*>(base + QNST * STAGE_BYTES + 64);   // FWD: 2 x [bias | gamma' | beta] of a tile's 128 columns

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    const int tiles_n = (N + QBN - 1) / QBN, tiles_m = (M + QBM - 1) / QBM;
    const int ntiles = tiles_n * tiles_m * nsplit;
    // k-blocks of one tile: FWD / STORE walk the segments (each padded to whole k-blocks by TMA zero fill), WGRAD walks its split
    int nkb_all = 0;
    for (int s = 0; s < segs.n; ++s) nkb_all += (segs.k[s] + QBK - 1) / QBK;
    auto tile_range = [&](int tile, int& m0, int& n0, int& z, int& kbeg, int& nkb) {
        z = tile / (tiles_n * tiles_m);
        int r = tile % (tiles_n * tiles_m);
        m0 = (r / tiles_n) * QBM;
        n0 = (r % tiles_n) * QBN;
        kbeg = 0;
        nkb = nkb_all;
        if (MODE == EPI_WGRAD) {
            kbeg = z * ksplit_len;
            int kend = min(ktot, kbeg + ksplit_len);
            nkb = kend > kbeg ? (kend - kbeg + QBK - 1) / QBK : 0;
        }
    };

    if (threadIdx.x == 0) {
        for (int s = 0; s < QNST; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }       // empty: one arrival per consumer warp
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------------ TMA producer
        reg_dealloc<40>();
        PROBE(0);
        if (warp == 0 && lane == 0) {
            int g = 0;
            for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
                int m0, n0, z, kbeg, nkb;
                tile_range(tile, m0, n0, z, kbeg, nkb);
                int seg = 0, kin = 0;                            // current segment, k offset inside it
                for (int kb = 0; kb < nkb; ++kb, ++g) {
                    const int s = g % QNST, it = g / QNST;
                    if (it > 0) mbar_wait(&empty[s], (it - 1) & 1);
                    int ka, kbcoord;
                    if (MODE == EPI_WGRAD) { ka = kbeg + kb * QBK; kbcoord = ka; }
                    else {
                        if (kin >= segs.k[seg]) { ++seg; kin = 0; }
                        ka = kin; kbcoord = segs.koff[seg] + kin;
                        kin += QBK;
                    }
                    mbar_expect_tx(&full[s], 2 * (A_BYTES + B_BYTES));
                    if (!A_MN) {
                        tma_load_2d(a_hi(s), &maps.a_hi[seg], &full[s], ka, m0);
                        tma_load_2d(a_lo(s), &maps.a_lo[seg], &full[s], ka, m0);
                    } else {
#pragma unroll
                        for (int i = 0; i < QBM / 64; ++i) {
                            tma_load_2d(a_hi(s) + i * 8192, &maps.a_hi[seg], &full[s], m0 + 64 * i, ka);
                            tma_load_2d(a_lo(s) + i * 8192, &maps.a_lo[seg], &full[s], m0 + 64 * i, ka);
                        }
                    }
                    if (!B_MN) {
                        tma_load_2d(b_hi(s), &maps.b_hi, &full[s], kbcoord, n0);
                        tma_load_2d(b_lo(s), &maps.b_lo, &full[s], kbcoord, n0);
                    } else {
#pragma unroll
                        for (int i = 0; i < QBN / 64; ++i) {
                            tma_load_2d(b_hi(s) + i * 8192, &maps.b_hi, &full[s], n0 + 64 * i, kbcoord);
                            tma_load_2d(b_lo(s) + i * 8192, &maps.b_lo, &full[s], n0 + 64 * i, kbcoord);
                        }
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ consumers: warp group cw owns rows [64 cw, 64 cw + 64)
        reg_alloc<232>();
        const int cw = wg - 1, cwarp = warp - 4;
        constexpr uint32_t a_step = A_MN ? 2048u : 32u, b_step = B_MN ? 2048u : 32u;   // bytes per 16-element k-step
        constexpr int TA = A_MN ? 1 : 0, TB = B_MN ? 1 : 0;
        float d[QBN / 2];
        int g = 0, use = 0;
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            int m0, n0, z, kbeg, nkb;
            tile_range(tile, m0, n0, z, kbeg, nkb);
            if (nkb == 0) {
#pragma unroll
                for (int i = 0; i < QBN / 2; ++i) d[i] = 0.f;
            }
            // FWD: the 384 per-column epilogue constants of this tile (bias, gamma * 1/sqrt(1 + eps), beta; each consumer thread
            // fetches v = ct and ct + 256) are loaded now, so their latency hides under the main loop, and handed over through
            // shared memory after it
            const int ct = threadIdx.x - 128;
            float pre[2] = {0.f, 0.f};
            if (MODE == EPI_FWD) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int v = ct + 256 * i, c = n0 + (v & 127);
                    const bool in = c < ep.n_logical;
                    if (v < 128) pre[i] = in ? __ldg(ep.bias + c) : 0.f;
                    else if (v < 256) pre[i] = (in && ep.bn) ? __ldg(ep.gamma + c) * 0.99950037468777f : 1.f;
                    else if (v < 384) pre[i] = (in && ep.bn) ? __ldg(ep.beta + c) : 0.f;
                }
            }
            int prev = -1;
            for (int kb = 0; kb < nkb; ++kb, ++g) {
                const int s = g % QNST, it = g / QNST;
                mbar_wait(&full[s], it & 1);
                if (g == 0) PROBE(1);
                const uint32_t sa_hi = smem_u32(a_hi(s)) + cw * 8192, sa_lo = smem_u32(a_lo(s)) + cw * 8192;   // 64 rows (or one 64-column box) per group
                const uint32_t sb_hi = smem_u32(b_hi(s)), sb_lo = smem_u32(b_lo(s));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < QBK / 16; ++k) {
                    const uint64_t da_hi = A_MN ? make_desc_mn(sa_hi + k * a_step) : make_desc(sa_hi + k * a_step);
                    const uint64_t da_lo = A_MN ? make_desc_mn(sa_lo + k * a_step) : make_desc(sa_lo + k * a_step);
                    const uint64_t db_hi = B_MN ? make_desc_mn(sb_hi + k * b_step) : make_desc(sb_hi + k * b_step);
                    const uint64_t db_lo = B_MN ? make_desc_mn(sb_lo + k * b_step) : make_desc(sb_lo + k * b_step);
                    wgmma_bf16<TA, TB>(d, da_lo, db_hi, (kb > 0 || k > 0) ? 1u : 0u);
                    wgmma_bf16<TA, TB>(d, da_hi, db_lo, 1u);
                    wgmma_bf16<TA, TB>(d, da_hi, db_hi, 1u);
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
            if (cwarp == 0) PROBE(use == 0 ? 2 : 3);
            // two buffers by tile parity: a thread writes tile t + 2's constants only after the barrier of tile t + 1, which every
            // consumer thread reaches after its epilogue of tile t
            const float* ev = epi_vec + (use & 1) * 384;
            if (MODE == EPI_FWD) {
                epi_vec[(use & 1) * 384 + ct] = pre[0];
                if (ct < 128) epi_vec[(use & 1) * 384 + ct + 256] = pre[1];
                bar_sync(1, 256);                                 // the two consumer warp groups
            }

            // ---- epilogue from the accumulator fragment: rows r0 and r0 + 8, columns n0 + 8 j + 2 (lane % 4) + {0, 1}
            const int r0 = m0 + cw * 64 + (warp & 3) * 16 + (lane >> 2);
            const int cq = 2 * (lane & 3);
            // The activation is dispatched once per tile, not per element: the relu body is then straight-line code the compiler
            // can schedule across column groups (loads of the next group's bias / gamma / beta under the current group's stores).
            auto epilogue = [&](auto relu) {
                constexpr bool RELU = decltype(relu)::value;
                uint32_t qh[2][2] = {}, ql[2][2] = {};          // FWD: bf16 hi / lo pairs of groups j - 1 and j, rows r0 and r0 + 8
#pragma unroll
                for (int j = 0; j < QBN / 8; ++j) {
                    const int c = n0 + 8 * j + cq;
                    if (n0 + 8 * j < N) {
                        if (MODE == EPI_FWD) {
                            const bool in0 = c < ep.n_logical, in1 = c + 1 < ep.n_logical;
                            const int cl = 8 * j + cq;                   // column inside the tile
                            const float b0 = ev[cl], b1 = ev[cl + 1], g0 = ev[128 + cl], g1 = ev[129 + cl], e0 = ev[256 + cl], e1 = ev[257 + cl];
#pragma unroll
                            for (int hh = 0; hh < 2; ++hh) {
                                const int r = r0 + 8 * hh;
                                if (r >= M) continue;
                                const bool rv = r < ep.m_valid;          // rows past the batch: zeros
                                float a0 = 0.f, a1 = 0.f, h0 = 0.f, h1 = 0.f;
                                if (rv && in0) { a0 = RELU ? fmaxf(d[4 * j + 2 * hh] + b0, 0.f) : act_fwd(ep.act, d[4 * j + 2 * hh] + b0); h0 = fmaf(a0, g0, e0); }
                                if (rv && in1) { a1 = RELU ? fmaxf(d[4 * j + 2 * hh + 1] + b1, 0.f) : act_fwd(ep.act, d[4 * j + 2 * hh + 1] + b1); h1 = fmaf(a1, g1, e1); }
                                const int64_t o = (int64_t)r * ep.ldh + c;
                                if (ep.A_out != ep.H_out) *reinterpret_cast<float2*>(ep.A_out + o) = make_float2(a0, a1);
                                if (ep.H_out) *reinterpret_cast<float2*>(ep.H_out + o) = make_float2(h0, h1);   // fp32 copy only where something reads it
                                split_pair(h0, h1, qh[j & 1][hh], ql[j & 1][hh]);
                            }
                            // The bf16 copies of groups j - 1 and j leave together: lane q of a quad gathers columns 16 (j / 2) + 4 q
                            // to + 3 (two pairs from lanes 2 (q % 2) and 2 (q % 2) + 1 of group j - 1 + q / 2), so every store writes
                            // a whole 32-byte sector instead of half of one.  N is a multiple of 32, so both groups are in range.
                            if (j & 1) {
                                const int q = lane & 3, src = (lane & ~3) + 2 * (q & 1);
                                const int64_t cp = n0 + 16 * (j >> 1) + 4 * q;
#pragma unroll
                                for (int hh = 0; hh < 2; ++hh) {
                                    uint2 vh, vl;
                                    const uint32_t h0a = __shfl_sync(0xffffffffu, qh[0][hh], src), h1a = __shfl_sync(0xffffffffu, qh[1][hh], src);
                                    const uint32_t h0b = __shfl_sync(0xffffffffu, qh[0][hh], src + 1), h1b = __shfl_sync(0xffffffffu, qh[1][hh], src + 1);
                                    const uint32_t l0a = __shfl_sync(0xffffffffu, ql[0][hh], src), l1a = __shfl_sync(0xffffffffu, ql[1][hh], src);
                                    const uint32_t l0b = __shfl_sync(0xffffffffu, ql[0][hh], src + 1), l1b = __shfl_sync(0xffffffffu, ql[1][hh], src + 1);
                                    vh.x = q < 2 ? h0a : h1a; vh.y = q < 2 ? h0b : h1b;
                                    vl.x = q < 2 ? l0a : l1a; vl.y = q < 2 ? l0b : l1b;
                                    const int r = r0 + 8 * hh;
                                    if (r >= M) continue;
                                    const int64_t o = (int64_t)r * ep.ldh + cp;
                                    *reinterpret_cast<uint2*>(ep.Hs_hi + o) = vh;
                                    *reinterpret_cast<uint2*>(ep.Hs_lo + o) = vl;
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
            };
            if (MODE == EPI_FWD && ep.act == WD_ACT_RELU) epilogue(std::true_type{});
            else epilogue(std::false_type{});
            if (cwarp == 0) PROBE(use == 0 ? 4 : 5);
            ++use;
        }
    }
}

int g_probe_slot = 0;

template <int MODE>
int launch_q(WdModel* m, const QMaps& maps, const QSegs& segs, int M, int N, int ktot, int splits, int ksplit_len, const Epi& ep) {
    constexpr int smem = QNST * 2 * (QBM * 128 + QBN * 128) + 1024 + 64 + 2 * 384 * 4;
    static bool configured = false;
    static int num_sms = 0;
    if (!configured) {
        WD_CUDA(cudaFuncSetAttribute(tc_gemm_bf16_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        WD_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, m->device));
        configured = true;
    }
    const int nsplit = MODE == EPI_WGRAD ? splits : 1;
    const int ntiles = ((N + QBN - 1) / QBN) * ((M + QBM - 1) / QBM) * nsplit;
    static const bool probe_on = getenv("WD_GEMM_PROBE") != nullptr;
    const int probe = probe_on ? (g_probe_slot++ & 31) : -1;
    tc_gemm_bf16_kernel<MODE><<<ntiles < num_sms ? ntiles : num_sms, Q_THREADS, smem, m->stream>>>(maps, segs, M, N, ktot, ksplit_len, nsplit, ep, probe);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

}  // namespace

// debugging aid (not part of the public header): copies the probe stamps of the last 32 launches, resets the slot counter
extern "C" int wd_debug_gemm_probe(unsigned long long* out) {
    cudaDeviceSynchronize();
    cudaError_t e = cudaMemcpyFromSymbol(out, g_probe, sizeof(unsigned long long) * 32 * 8);
    g_probe_slot = 0;
    return e == cudaSuccess ? 0 : -1;
}

int tc_gemm_bf16(WdModel* m, int mode, const GemmA& A, const GemmB& B, int M, int N, const Epi& ep, int splits, int ksplit_len) {
    constexpr CUtensorMapDataType BF16 = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    if (N % 32 != 0 || A.n > kMaxSegs || !B.hi || !B.lo) { set_error("bf16 GEMM engine: unsupported operands"); return WD_EUNSUPPORTED; }
    QMaps maps;
    QSegs segs{};
    segs.n = A.n;
    int rc, ktot = 0;
    const bool a_mn = mode == EPI_WGRAD, b_mn = mode == EPI_FWD || mode == EPI_WGRAD;
    for (int s = 0; s < A.n; ++s) {
        if (!A.hi[s] || !A.lo[s]) { set_error("bf16 GEMM engine: operand without hi/lo copies"); return WD_EINVAL; }
        // K-major: [M rows][k contiguous], box 64 k x 128 rows.  MN-major: [k rows][M contiguous], box 64 columns x 64 k-rows
        if (!a_mn) {
            if ((rc = make_tensor_map(&maps.a_hi[s], BF16, A.hi[s], M, A.k[s], A.ld[s], QBM))) return rc;
            if ((rc = make_tensor_map(&maps.a_lo[s], BF16, A.lo[s], M, A.k[s], A.ld[s], QBM))) return rc;
        } else {
            if ((rc = make_tensor_map(&maps.a_hi[s], BF16, A.hi[s], A.k[s], M, A.ld[s], 64))) return rc;
            if ((rc = make_tensor_map(&maps.a_lo[s], BF16, A.lo[s], A.k[s], M, A.ld[s], 64))) return rc;
        }
        segs.k[s] = A.k[s]; segs.koff[s] = ktot;
        ktot += A.k[s];
    }
    for (int s = A.n; s < kMaxSegs; ++s) { maps.a_hi[s] = maps.a_hi[0]; maps.a_lo[s] = maps.a_lo[0]; }
    if (!b_mn) {
        if ((rc = make_tensor_map(&maps.b_hi, BF16, B.hi, N, ktot, B.ld, QBN))) return rc;
        if ((rc = make_tensor_map(&maps.b_lo, BF16, B.lo, N, ktot, B.ld, QBN))) return rc;
    } else {
        if ((rc = make_tensor_map(&maps.b_hi, BF16, B.hi, ktot, N, B.ld, 64))) return rc;
        if ((rc = make_tensor_map(&maps.b_lo, BF16, B.lo, ktot, N, B.ld, 64))) return rc;
    }
    if (mode == EPI_WGRAD) ksplit_len = (ksplit_len + QBK - 1) / QBK * QBK;
    if (mode == EPI_FWD && (!ep.Hs_hi || !ep.Hs_lo)) { set_error("bf16 GEMM engine: epilogue without hi/lo outputs"); return WD_EINVAL; }
    if (mode == EPI_FWD) return launch_q<EPI_FWD>(m, maps, segs, M, N, ktot, splits, ksplit_len, ep);
    if (mode == EPI_STORE) return launch_q<EPI_STORE>(m, maps, segs, M, N, ktot, splits, ksplit_len, ep);
    return launch_q<EPI_WGRAD>(m, maps, segs, M, N, ktot, splits, ksplit_len, ep);
}

}  // namespace wd
