// Dense half of the step: the Dnn / ResDnn / DenseDnn towers, the binary head, their backward and the
// dense optimizers.
//
//   layer forward    act(x W + b) -> [BN inference affine] -> concat          (reference dnn.py:92-233, SURVEY A.8)
//   head             logits = sum of tower logits + wide logit; sigmoid CE, SUM (reference joint.py:216-222, 402-406)
//   backward         MatMul grads, activation / affine grads                  (reference joint.py:234-239 minimize())
//   dense optimizer  ApplyAdagrad / ApplyFtrl / SGD with constant LR (Q1)     (reference model_util.py:62-105)
//
// Every matrix product is a GEMM  C[M,N] = sum_k A[M,k] * B[k,N]  over a GemmA (up to kMaxSegs input segments) and a GemmB.
// Each engine reads its operands from stored copies of one operand family (WdModel::operands, decided in wd_model_create), and a
// model allocates and writes only its family's copies:
//
//                fp32 family: ffma, tc1x, tc3x                        bf16 family: bf16x3
//                fp32, both operands K-contiguous ("TN")              bf16 hi / lo copies (GemmA::hi / lo, GemmB::hi / lo)
//   forward  A   X0 / H [B, K] input segments                         X0s / Hs [B, K]                        K-major
//            B   Wt [N, K]           (tc3x: tf32 splits Wt_hi / Wt_lo)   Wq [K, N]                           MN-major
//   dgrad    A   dZ [B, N]                                            dZs [B, N]                             K-major
//            B   W [K, N] rows of one input segment (tc3x: W_hi / W_lo)  Wq rows of the segment             K-major
//   wgrad    A   X0T / HT [K, ldt], reduction over the batch padded   X0s / Hs [B, K], reduction over B      MN-major
//            B   dZT [N, ldt]        to 16 (split over the batch)     dZs [B, N]                             MN-major
//   written by   the forward epilogue (H, HT), transpose_kernel        the forward epilogue (Hs), x0_split_kernel (X0s),
//                (X0T), act_bn_bwd_kernel (dZ, dZT),                   act_bn_bwd_q_kernel / logits_act_bwd_q_kernel (dZs),
//                dense_apply_kernel (Wt and the tf32 splits)           dense_vec_kernel (Wq)
// Both families keep the post-activation values A and the gradients dH in fp32.  The bf16 family keeps the layer output H in
// fp32 only for layers the logits layer reads (logits_head_kernel and the logits backward are not GEMMs).  fwd_operands,
// dgrad_operands and wgrad_operands fill GemmA / GemmB from this table; the drivers mlp_forward / mlp_backward only choose
// between the family's named kernels.
//
// This file also holds the fp32 CUDA-core (FFMA) engine: exact fp32 products, the parity engine and the reference the tensor-core
// engines (tf32: gemm_tc.cu, bf16: gemm_bf16.cu) are validated against.
#include "common.cuh"
#include "gemm.cuh"

namespace wd {

constexpr int BM = 128, BN = 128, BK = 16, GT = 256;

template <int MODE>
__global__ void __launch_bounds__(GT) gemm_tn_ffma(GemmA A, const float* __restrict__ Bm, int ldb, int M, int N, int ksplit_len, Epi ep) {
    __shared__ __align__(16) float As[2][BK][BM + 4];
    __shared__ __align__(16) float Bs[2][BK][BN + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    // K range of this CTA (split over blockIdx.z in WGRAD); segments are walked in order
    int ktot = 0;
    for (int s = 0; s < A.n; ++s) ktot += A.k[s];
    int kbeg = 0, kend = ktot;
    if (MODE == EPI_WGRAD) {
        kbeg = blockIdx.z * ksplit_len;
        kend = min(ktot, kbeg + ksplit_len);
    }
    const int lrow = tid >> 2, lkc = tid & 3;          // load mapping: 64 rows x 4 k-chunks per pass, 2 passes
    float4 ra[2], rb[2];

    auto gload = [&](int kg) {                         // kg: global k (multiple of 16) in concatenated space
        int s = 0, kk = kg;
        while (s < A.n - 1 && kk >= A.k[s]) { kk -= A.k[s]; ++s; }
        const float* ap = A.ptr[s];
        const int lda = A.ld[s];
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            int r = lrow + p * 64;
            int gm = m0 + r, gn = n0 + r;
            ra[p] = (gm < M) ? *reinterpret_cast<const float4*>(ap + (int64_t)gm * lda + kk + lkc * 4) : make_float4(0, 0, 0, 0);
            rb[p] = (gn < N) ? *reinterpret_cast<const float4*>(Bm + (int64_t)gn * ldb + kg + lkc * 4) : make_float4(0, 0, 0, 0);
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            int r = lrow + p * 64;
            As[buf][lkc * 4 + 0][r] = ra[p].x; As[buf][lkc * 4 + 1][r] = ra[p].y;
            As[buf][lkc * 4 + 2][r] = ra[p].z; As[buf][lkc * 4 + 3][r] = ra[p].w;
            Bs[buf][lkc * 4 + 0][r] = rb[p].x; Bs[buf][lkc * 4 + 1][r] = rb[p].y;
            Bs[buf][lkc * 4 + 2][r] = rb[p].z; Bs[buf][lkc * 4 + 3][r] = rb[p].w;
        }
    };

    int buf = 0;
    if (kbeg < kend) {
        gload(kbeg);
        sstore(0);
    }
    __syncthreads();
    for (int kg = kbeg; kg < kend; kg += BK) {
        bool more = kg + BK < kend;
        if (more) gload(kg + BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
            float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
            float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (more) sstore(buf ^ 1);
        __syncthreads();
        buf ^= 1;
    }

    // ---- epilogue: thread owns rows {ty*4+i, 64+ty*4+i}, cols {tx*4+j, 64+tx*4+j}
#pragma unroll
    for (int ih = 0; ih < 2; ++ih) {
#pragma unroll
        for (int jh = 0; jh < 2; ++jh) {
            const int mb = m0 + ih * 64 + ty * 4, nb = n0 + jh * 64 + tx * 4;
            if (nb >= N) continue;
            if (MODE == EPI_FWD) {
                float hv[4][4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int gm = mb + i;
                    float a4[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int gn = nb + j;
                        float a = 0.f, h = 0.f;
                        if (gn < ep.n_logical && gm < ep.m_valid) {
                            a = act_fwd(ep.act, acc[ih * 4 + i][jh * 4 + j] + ep.bias[gn]);
                            h = bn_out(a, ep.gamma, ep.beta, gn, ep.bn);
                        }
                        a4[j] = a;
                        hv[i][j] = h;
                    }
                    if (gm < M) {
                        if (ep.A_out != ep.H_out)
                            *reinterpret_cast<float4*>(ep.A_out + (int64_t)gm * ep.ldh + nb) = make_float4(a4[0], a4[1], a4[2], a4[3]);
                        *reinterpret_cast<float4*>(ep.H_out + (int64_t)gm * ep.ldh + nb) = make_float4(hv[i][0], hv[i][1], hv[i][2], hv[i][3]);
                    }
                }
                if (ep.HT) {
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        *reinterpret_cast<float4*>(ep.HT + (int64_t)(nb + j) * ep.ldt + mb) = make_float4(hv[0][j], hv[1][j], hv[2][j], hv[3][j]);
                }
            } else {
                float* Cb = ep.C + (MODE == EPI_WGRAD ? (int64_t)blockIdx.z * ep.split_stride : 0);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int gm = mb + i;
                    if (gm >= M) continue;
                    float4 v = make_float4(acc[ih * 4 + i][jh * 4 + 0], acc[ih * 4 + i][jh * 4 + 1], acc[ih * 4 + i][jh * 4 + 2], acc[ih * 4 + i][jh * 4 + 3]);
                    float4* dst = reinterpret_cast<float4*>(Cb + (int64_t)gm * ep.ldc + nb);
                    if (MODE == EPI_STORE && ep.accumulate) {
                        float4 o = *dst;
                        v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
                    }
                    *dst = v;
                }
            }
        }
    }
}

static void launch_gemm(WdModel* m, int mode, const GemmA& A, const GemmB& B, int M, int N, const Epi& ep, int splits, int ksplit_len) {
    dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM, mode == EPI_WGRAD ? splits : 1);
    if (mode == EPI_FWD) gemm_tn_ffma<EPI_FWD><<<grid, GT, 0, m->stream>>>(A, B.ptr, B.ld, M, N, 0, ep);
    else if (mode == EPI_STORE) gemm_tn_ffma<EPI_STORE><<<grid, GT, 0, m->stream>>>(A, B.ptr, B.ld, M, N, 0, ep);
    else gemm_tn_ffma<EPI_WGRAD><<<grid, GT, 0, m->stream>>>(A, B.ptr, B.ld, M, N, ksplit_len, ep);
    m->launches++;
}

static int run_gemm(WdModel* m, int mode, const GemmA& A, const GemmB& B, int M, int N, const Epi& ep, int splits = 1, int ksplit_len = 0) {
    static const char* kNamesL[3][4] = {{"gemm_fwd_l0", "gemm_fwd_l1", "gemm_fwd_l2", "gemm_fwd_l3+"},
                                        {"gemm_dgrad_l0", "gemm_dgrad_l1", "gemm_dgrad_l2", "gemm_dgrad_l3+"},
                                        {"gemm_wgrad_l0", "gemm_wgrad_l1", "gemm_wgrad_l2", "gemm_wgrad_l3+"}};
    const char* kNames[3] = {kNamesL[0][m->cur_layer < 3 ? m->cur_layer : 3], kNamesL[1][m->cur_layer < 3 ? m->cur_layer : 3],
                             kNamesL[2][m->cur_layer < 3 ? m->cur_layer : 3]};
    mark(m, "mlp_other");
    if (m->operands == kBf16Operands) {
        int rc = tc_gemm_bf16(m, mode, A, B, M, N, ep, splits, ksplit_len);
        mark(m, kNames[mode]);
        return rc;
    }
    if (m->gemm_engine == WD_GEMM_TC3X || m->gemm_engine == WD_GEMM_TC1X) {
        int rc = tc_gemm(m, mode, A, B, M, N, ep, splits, ksplit_len);
        if (rc != WD_EUNSUPPORTED) { mark(m, kNames[mode]); return rc; }
        m->gemm_fallbacks++;                              // loud: counted, reported by wd_gemm_fallback_count, asserted 0 in the tests
        static bool warned = false;
        if (!warned) { fprintf(stderr, "libwd_b200: wgmma engine does not cover a GEMM (M=%d N=%d segs=%d): running it on the FFMA kernel\n", M, N, A.n); warned = true; }
    }
    launch_gemm(m, mode, A, B, M, N, ep, splits, ksplit_len);
    mark(m, kNames[mode]);
    return WD_OK;
}

// --------------------------------------------------------------------------------------- small kernels
// out[n][m] = in[m][n] for m < M (zeros for M <= m < Mpad), 32x32 tiles through shared memory
__global__ void transpose_kernel(const float* __restrict__ in, int ld_in, int M, int Mpad, int N, float* __restrict__ out, int ld_out) {
    __shared__ float t[32][33];
    int m0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += 8) {
        int mm = m0 + i, nn = n0 + threadIdx.x;
        t[i][threadIdx.x] = (mm < M && nn < N) ? in[(int64_t)mm * ld_in + nn] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        int nn = n0 + i, mm = m0 + threadIdx.x;
        if (nn < N && mm < Mpad) out[(int64_t)nn * ld_out + mm] = t[threadIdx.x][i];
    }
}

// 3xBF16 engine: bf16 hi / lo copies of the deep input [M, ld] (the only form the tensor-core GEMMs read)
__global__ void x0_split_kernel(const float* __restrict__ in, int64_t n4, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 x = reinterpret_cast<const float4*>(in)[i];
        store_split4(hi + 4 * i, lo + 4 * i, x.x, x.y, x.z, x.w);
    }
}

// dropout of a hidden layer (rare path, unfused): the forward GEMM's epilogue left the post-activation values A; this kernel
// rebuilds the layer output from them with the keep mask: H = [BN affine](A * mask / keep) and its bf16 hi / lo or transposed copies
__global__ void __launch_bounds__(256) dropout_fwd_kernel(int B, int N, int n_logical, const float* __restrict__ A, int ld,
                                                         const float* __restrict__ gamma, const float* __restrict__ beta, int bn,
                                                         float* __restrict__ H, __nv_bfloat16* __restrict__ q_hi, __nv_bfloat16* __restrict__ q_lo,
                                                         float* __restrict__ HT, int ldt, DropArgs dr) {
    const unsigned long long key = drop_key(dr);
    const float inv_keep = 1.f / (1.f - dr.rate);
    const int64_t total = (int64_t)B * N;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int mrow = (int)(t / N), n = (int)(t % N);
        float h = 0.f;
        if (n < n_logical) {
            const float a = A[(int64_t)mrow * ld + n] * drop_mult(key, dr.row0 + (unsigned)mrow, (unsigned)n, dr.rate, inv_keep);
            h = bn_out(a, gamma, beta, n, bn);
        }
        if (H) H[(int64_t)mrow * ld + n] = h;
        if (q_hi) {
            __nv_bfloat16 hh, hl;
            split_bf16(h, hh, hl);
            q_hi[(int64_t)mrow * ld + n] = hh; q_lo[(int64_t)mrow * ld + n] = hl;
        }
        if (HT) HT[(int64_t)n * ldt + mrow] = h;
    }
}

// input segments of a tower's logits layer
struct GemvSegs { int n; const float* ptr[kMaxSegs]; int ld[kMaxSegs]; int k[kMaxSegs]; int koff[kMaxSegs]; };

// ---- head: logits layers of all towers (one warp per example) + wide logit + sigmoid cross entropy + dlogit + the batch loss
// (block partials, summed in block order by the last block to finish), in one launch
struct HeadIn { int n; GemvSegs S[kMaxTowers]; const float* kernel[kMaxTowers]; const float* bias[kMaxTowers]; float* tower_logit[kMaxTowers]; };
__global__ void __launch_bounds__(256) logits_head_kernel(HeadIn in, int B, const float* __restrict__ wide_logit, const float* __restrict__ label,
                                                        const float* __restrict__ weight, float* __restrict__ logits, float* __restrict__ dlogit,
                                                        float* __restrict__ loss_part, int32_t* __restrict__ counter, float* __restrict__ loss_out) {
    __shared__ float red[8];
    __shared__ bool is_last;
    // eight lanes per example, four examples per warp: a lane's loads (up to four 16-byte loads per segment round) are all in
    // flight before the first one is used
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, lig = lane & 7, grp = lane >> 3;
    const int nw = (gridDim.x * blockDim.x) >> 5;
    float lsum = 0.f;
    for (int b0 = warp * 4; b0 < B; b0 += nw * 4) {
        const int b = b0 + grp;
        const bool live = b < B;
        float x = (live && wide_logit) ? wide_logit[b] : 0.f;
        for (int t = 0; t < in.n; ++t) {
            const GemvSegs& S = in.S[t];
            float acc = 0.f;
            if (live) {
                for (int s = 0; s < S.n; ++s) {
                    const float* row = S.ptr[s] + (int64_t)b * S.ld[s];
                    const float* kw = in.kernel[t] + S.koff[s];
                    const int K = S.k[s];
                    int k = lig * 4;
                    for (; k + 96 < K; k += 128) {
                        float4 xv[4], w[4];
#pragma unroll
                        for (int u = 0; u < 4; ++u) { xv[u] = *reinterpret_cast<const float4*>(row + k + 32 * u); w[u] = *reinterpret_cast<const float4*>(kw + k + 32 * u); }
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            acc = fmaf(xv[u].x, w[u].x, acc); acc = fmaf(xv[u].y, w[u].y, acc); acc = fmaf(xv[u].z, w[u].z, acc); acc = fmaf(xv[u].w, w[u].w, acc);
                        }
                    }
                    for (; k < K; k += 32) {
                        const float4 xv = *reinterpret_cast<const float4*>(row + k);
                        const float4 w = *reinterpret_cast<const float4*>(kw + k);
                        acc = fmaf(xv.x, w.x, acc); acc = fmaf(xv.y, w.y, acc); acc = fmaf(xv.z, w.z, acc); acc = fmaf(xv.w, w.w, acc);
                    }
                }
            }
#pragma unroll
            for (int d = 4; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
            const float tl = acc + in.bias[t][0];
            if (lig == 0 && live) in.tower_logit[t][b] = tl;
            x += tl;
        }
        if (lig == 0 && live) {
            logits[b] = x;
            if (label) {
                const float y = label[b], w = weight ? weight[b] : 1.f;
                lsum += w * (fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x))));      // sigmoid cross entropy with logits (SURVEY A.10)
                if (dlogit) dlogit[b] = (1.f / (1.f + expf(-x)) - y) * w;
            }
        }
    }
    lsum += __shfl_xor_sync(0xffffffffu, lsum, 8);                     // the warp's four examples, fixed order
    lsum += __shfl_xor_sync(0xffffffffu, lsum, 16);
    if (lane == 0) red[threadIdx.x >> 5] = lsum;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < 8; ++i) s += red[i];
        loss_part[blockIdx.x] = s;
        __threadfence();
        is_last = atomicAdd(counter, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (is_last) {                                                    // fixed-order tree over the block partials (<= 512): deterministic
        __shared__ double dred[256];
        __threadfence();
        const int nb = (int)gridDim.x;
        double s = 0.0;
        for (int i = threadIdx.x; i < nb; i += 256) s += (double)__ldcg(loss_part + i);
        dred[threadIdx.x] = s;
        __syncthreads();
        for (int d = 128; d > 0; d >>= 1) {
            if ((int)threadIdx.x < d) dred[threadIdx.x] += dred[threadIdx.x + d];
            __syncthreads();
        }
        if (threadIdx.x == 0) { *loss_out = (float)dred[0]; *counter = 0; }
    }
}

// ---- fused logits-layer backward for one input segment: weight-gradient partials per 128-row tile, the data gradient of the
// segment, and (first segment) the bias partial — which is also the wide bias's gradient partial (both are sums of dlogit)
__global__ void __launch_bounds__(256) logits_bwd_kernel(int B, int K, const float* __restrict__ src, int ld, const float* __restrict__ dlogit,
                                                        const float* __restrict__ kw, float* __restrict__ gpart, int64_t gstride,
                                                        float* __restrict__ bias_part, int64_t bias_stride, float* __restrict__ wide_bias_part,
                                                        int64_t wide_bias_stride, float* __restrict__ dst, int dld, int accumulate) {
    __shared__ float red[4][64];
    __shared__ float dl[128];
    const int rt = blockIdx.y, kx = threadIdx.x & 63, ry = threadIdx.x >> 6;
    const int k = blockIdx.x * 64 + kx;
    const int b0 = rt * 128;
    if (threadIdx.x < 128) dl[threadIdx.x] = (b0 + threadIdx.x < B) ? dlogit[b0 + threadIdx.x] : 0.f;
    __syncthreads();
    float acc = 0.f;
    if (k < K) {
        const int r0 = b0 + ry * 32;
        const float w = dst ? kw[k] : 0.f;
#pragma unroll 8
        for (int i = 0; i < 32; ++i)
            if (r0 + i < B) {
                const float g = dl[ry * 32 + i];
                acc = fmaf(src[(int64_t)(r0 + i) * ld + k], g, acc);
                if (dst) {
                    float* d = dst + (int64_t)(r0 + i) * dld + k;
                    *d = accumulate ? *d + g * w : g * w;
                }
            }
    }
    red[ry][kx] = acc;
    __syncthreads();
    if (ry == 0 && k < K) gpart[(int64_t)rt * gstride + k] = red[0][kx] + red[1][kx] + red[2][kx] + red[3][kx];
    if (blockIdx.x == 0 && threadIdx.x == 0 && (bias_part || wide_bias_part)) {
        float s = 0.f;
        for (int i = 0; i < 128; ++i) s += dl[i];
        if (bias_part) bias_part[(int64_t)rt * bias_stride] = s;
        if (wide_bias_part) wide_bias_part[(int64_t)rt * wide_bias_stride] = s;
    }
}

// hidden layer backward through [BN affine] and activation:
//   da = dH * gamma/sqrt(1+eps); dZ = da * act'(a); column partial sums of dZ (bias), dH*a/sqrt(1+eps) (gamma), dH (beta)
// block = 32 columns x 128 rows (one row tile); writes dZ and dZT (zero padded to the tile)
__global__ void __launch_bounds__(256) act_bn_bwd_kernel(int B, int N, int n_logical, const float* __restrict__ dH, const float* __restrict__ Aact,
                                                        int ld, const float* __restrict__ gamma, int act, int bn,
                                                        float* __restrict__ dZ, float* __restrict__ dZT, int ldt,
                                                        float* __restrict__ p_bias, float* __restrict__ p_gamma, float* __restrict__ p_beta,
                                                        int64_t pstride, DropArgs dr) {
    __shared__ float tile[32][33];
    const unsigned long long dkey = dr.rate > 0.f ? drop_key(dr) : 0ull;
    const float inv_keep = dr.rate > 0.f ? 1.f / (1.f - dr.rate) : 1.f;
    __shared__ float red[3][8][32];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;       // 32 x 8
    const int n = blockIdx.x * 32 + tx, rt = blockIdx.y;
    const float inv = 0.99950037468777f;
    float sb = 0.f, sg = 0.f, sbe = 0.f;
    const float gsc = (bn && n < n_logical) ? gamma[n] * inv : 1.f;
    for (int sub = 0; sub < 4; ++sub) {                           // 4 sub-tiles of 32 rows
        const int mbase = rt * 128 + sub * 32;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int mm = mbase + ty * 4 + i;
            float dz = 0.f;
            if (mm < B && n < n_logical) {
                float dh = dH[(int64_t)mm * ld + n], a = Aact[(int64_t)mm * ld + n];
                const float dm = dr.rate > 0.f ? drop_mult(dkey, dr.row0 + (unsigned)mm, (unsigned)n, dr.rate, inv_keep) : 1.f;
                dz = dh * gsc * dm * act_bwd(act, a);
                sb += dz; sg += dh * (a * dm) * inv; sbe += dh;
            }
            if (mm < B && n < N) dZ[(int64_t)mm * ld + n] = dz;
            tile[ty * 4 + i][tx] = dz;
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int nn = blockIdx.x * 32 + ty * 4 + i;
            if (nn < N) dZT[(int64_t)nn * ldt + mbase + tx] = tile[tx][ty * 4 + i];
        }
        __syncthreads();
    }
    red[0][ty][tx] = sb; red[1][ty][tx] = sg; red[2][ty][tx] = sbe;
    __syncthreads();
    if (ty == 0 && n < N) {
        float a = 0.f, b = 0.f, c = 0.f;
        for (int i = 0; i < 8; ++i) { a += red[0][i][tx]; b += red[1][i][tx]; c += red[2][i][tx]; }
        p_bias[(int64_t)rt * pstride + n] = a;
        if (bn) { p_gamma[(int64_t)rt * pstride + n] = b; p_beta[(int64_t)rt * pstride + n] = c; }
    }
}

// The same for the 3xBF16 engine (dZ leaves as bf16 hi / lo copies only, no transposed copy): a block covers one 128-row tile x
// 64 columns; a thread owns 4 consecutive columns and every 16th row, and issues all sixteen 16-byte loads (dH and A of its 8
// rows) before the first use; 8-byte stores of the bf16 copies; the column partial sums go through shared memory in a fixed order.
__global__ void __launch_bounds__(256) act_bn_bwd_q_kernel(int B, int N, int n_logical, const float* __restrict__ dH, const float* __restrict__ Aact,
                                                          int ld, const float* __restrict__ gamma, int act, int bn,
                                                          float* __restrict__ p_bias, float* __restrict__ p_gamma, float* __restrict__ p_beta,
                                                          int64_t pstride, __nv_bfloat16* __restrict__ q_hi, __nv_bfloat16* __restrict__ q_lo, DropArgs dr) {
    __shared__ float red[3][16][64];
    const unsigned long long dkey = dr.rate > 0.f ? drop_key(dr) : 0ull;
    const float inv_keep = dr.rate > 0.f ? 1.f / (1.f - dr.rate) : 1.f;
    const int cx = threadIdx.x & 15, ry = threadIdx.x >> 4;
    const int n0 = blockIdx.x * 64 + cx * 4, rt = blockIdx.y, b0 = rt * 128;
    const float inv = 0.99950037468777f;
    float gsc[4], sb[4] = {0.f, 0.f, 0.f, 0.f}, sg[4] = {0.f, 0.f, 0.f, 0.f}, sbe[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 4; ++j) gsc[j] = (bn && n0 + j < n_logical) ? gamma[n0 + j] * inv : 1.f;
    if (n0 < N) {
        float4 dhv[8], av[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {                                  // rows past the batch re-read the last valid row
            const int mr = min(b0 + u * 16 + ry, B - 1);
            dhv[u] = *reinterpret_cast<const float4*>(dH + (int64_t)mr * ld + n0);
            av[u] = *reinterpret_cast<const float4*>(Aact + (int64_t)mr * ld + n0);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int mm = b0 + u * 16 + ry;
            if (mm >= B) continue;
            const float dh[4] = {dhv[u].x, dhv[u].y, dhv[u].z, dhv[u].w}, a[4] = {av[u].x, av[u].y, av[u].z, av[u].w};
            float dz[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                dz[j] = 0.f;
                if (n0 + j < n_logical) {
                    const float dm = dr.rate > 0.f ? drop_mult(dkey, dr.row0 + (unsigned)mm, (unsigned)(n0 + j), dr.rate, inv_keep) : 1.f;
                    dz[j] = dh[j] * gsc[j] * dm * act_bwd(act, a[j]);
                    sb[j] += dz[j]; sg[j] += dh[j] * (a[j] * dm) * inv; sbe[j] += dh[j];
                }
            }
            store_split4(q_hi + (int64_t)mm * ld + n0, q_lo + (int64_t)mm * ld + n0, dz[0], dz[1], dz[2], dz[3]);
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { red[0][ry][cx * 4 + j] = sb[j]; red[1][ry][cx * 4 + j] = sg[j]; red[2][ry][cx * 4 + j] = sbe[j]; }
    __syncthreads();
    if (threadIdx.x < 192) {
        const int which = threadIdx.x >> 6, c = threadIdx.x & 63, n = blockIdx.x * 64 + c;
        if (n < N && (which == 0 || bn)) {
            float x = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) x += red[which][i][c];
            (which == 0 ? p_bias : which == 1 ? p_gamma : p_beta)[(int64_t)rt * pstride + n] = x;
        }
    }
}

// 3xBF16 engine, last hidden layer of a tower whose only reader is the logits layer: the logits layer's backward (kernel / bias
// gradient partials, dH = dlogit x w) and the layer's own activation / batch-norm backward in ONE pass — dH never exists.
// Block = 128 rows x 64 columns, thread = 4 columns x 8 rows with all sixteen 16-byte loads (H and A) in flight before the first use;
// column partials through shared memory in a fixed order.
__global__ void __launch_bounds__(256) logits_act_bwd_q_kernel(int B, int N, int n_logical, const float* __restrict__ H, int ldh,
                                                              const float* __restrict__ Aact, int ld, const float* __restrict__ dlogit,
                                                              const float* __restrict__ kw, const float* __restrict__ gamma, int act, int bn,
                                                              float* __restrict__ p_kw, int64_t kw_stride, float* __restrict__ p_lbias, int64_t lbias_stride,
                                                              float* __restrict__ p_wbias, int64_t wbias_stride,
                                                              float* __restrict__ p_bias, float* __restrict__ p_gamma, float* __restrict__ p_beta, int64_t pstride,
                                                              __nv_bfloat16* __restrict__ q_hi, __nv_bfloat16* __restrict__ q_lo) {
    __shared__ float red[4][16][64];
    __shared__ float dl[128];
    const int cx = threadIdx.x & 15, ry = threadIdx.x >> 4;
    const int n0 = blockIdx.x * 64 + cx * 4, rt = blockIdx.y, b0 = rt * 128;
    const float inv = 0.99950037468777f;
    if (threadIdx.x < 128) dl[threadIdx.x] = (b0 + threadIdx.x < B) ? dlogit[b0 + threadIdx.x] : 0.f;
    float gsc[4], w[4], sk[4] = {0.f, 0.f, 0.f, 0.f}, sb[4] = {0.f, 0.f, 0.f, 0.f}, sg[4] = {0.f, 0.f, 0.f, 0.f}, sbe[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        gsc[j] = (bn && n0 + j < n_logical) ? gamma[n0 + j] * inv : 1.f;
        w[j] = n0 + j < N ? kw[n0 + j] : 0.f;
    }
    __syncthreads();
    if (n0 < N) {
        float4 hv[8], av[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {                                  // rows past the batch re-read the last valid row
            const int mr = min(b0 + u * 16 + ry, B - 1);
            hv[u] = *reinterpret_cast<const float4*>(H + (int64_t)mr * ldh + n0);
            av[u] = *reinterpret_cast<const float4*>(Aact + (int64_t)mr * ld + n0);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int mm = b0 + u * 16 + ry;
            if (mm >= B) continue;
            const float g = dl[u * 16 + ry];
            const float h[4] = {hv[u].x, hv[u].y, hv[u].z, hv[u].w}, a[4] = {av[u].x, av[u].y, av[u].z, av[u].w};
            float dz[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                sk[j] = fmaf(h[j], g, sk[j]);
                dz[j] = 0.f;
                if (n0 + j < n_logical) {
                    const float dh = g * w[j];
                    dz[j] = dh * gsc[j] * act_bwd(act, a[j]);
                    sb[j] += dz[j]; sg[j] += dh * a[j] * inv; sbe[j] += dh;
                }
            }
            store_split4(q_hi + (int64_t)mm * ld + n0, q_lo + (int64_t)mm * ld + n0, dz[0], dz[1], dz[2], dz[3]);
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { red[0][ry][cx * 4 + j] = sk[j]; red[1][ry][cx * 4 + j] = sb[j]; red[2][ry][cx * 4 + j] = sg[j]; red[3][ry][cx * 4 + j] = sbe[j]; }
    __syncthreads();
    {
        const int which = threadIdx.x >> 6, c = threadIdx.x & 63, n = blockIdx.x * 64 + c;      // 4 quantities x 64 columns
        if (n < N) {
            float x = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) x += red[which][i][c];
            if (which == 0) p_kw[(int64_t)rt * kw_stride + n] = x;
            else if (which == 1) p_bias[(int64_t)rt * pstride + n] = x;
            else if (bn) (which == 2 ? p_gamma : p_beta)[(int64_t)rt * pstride + n] = x;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && (p_lbias || p_wbias)) {
        float s = 0.f;
        for (int i = 0; i < 128; ++i) s += dl[i];
        if (p_lbias) p_lbias[(int64_t)rt * lbias_stride] = s;
        if (p_wbias) p_wbias[(int64_t)rt * wbias_stride] = s;
    }
}

// wide bias gradient partials: per 128-row tile sum of dlogit
__global__ void rowtile_sum_kernel(int B, const float* __restrict__ v, float* __restrict__ part, int64_t stride) {
    int rt = blockIdx.x;
    int b0 = rt * 128, b1 = min(B, b0 + 128);
    float s = 0.f;
    for (int b = b0 + threadIdx.x; b < b1; b += 32) s += v[b];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    if (threadIdx.x == 0) part[(int64_t)rt * stride] = s;
}
int wide_bias_grad(WdModel* m) {
    if (!m->use_wide) return WD_OK;
    if (m->use_deep && !m->towers.empty()) return WD_OK;               // written by the first logits_bwd_kernel launch of the step
    const int rts = (m->dbatch.B + 127) / 128;
    rowtile_sum_kernel<<<rts, 32, 0, m->stream>>>(m->dbatch.B, m->d_dlogit, m->d_gpart + m->dense[0].gpart_off, m->dense[0].gstride);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ---------------------------------------------------------------------------------- dense optimizer side
// G[i] = sum_p gpart[t.gpart_off + p * t.gstride + (i - t.off)] over the live partials of tensor t
__global__ void dense_reduce_kernel(const DenseTensor* __restrict__ T, int nt, int64_t total, const float* __restrict__ gpart,
                                    float* __restrict__ G, int live_row_tiles) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int lo = 0, hi = nt - 1;
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            if (T[mid].off <= i) lo = mid; else hi = mid - 1;
        }
        const DenseTensor t = T[lo];
        if (i - t.off >= t.count) { G[i] = 0.f; continue; }          // alignment gap between tensors
        int parts = t.g_rowtiles ? live_row_tiles : t.gparts;              // row-tile partials: only tiles of this batch
        float s = 0.f;
        const float* p = gpart + t.gpart_off + (i - t.off);
        for (int q = 0; q < parts; ++q) s += p[(int64_t)q * t.gstride];
        G[i] = s;
    }
}

struct OptParamsD { int kind; float lr, l1, l2, beta1, beta2, epsilon, rho, momentum; const float* bpow; };
static OptParamsD make_opt_d(const WdOptimizer& o, const float* bpow) {
    return OptParamsD{o.kind, o.lr, o.l1, o.l2, o.beta1, o.beta2, o.epsilon, o.rho, o.momentum, bpow};
}
__device__ __forceinline__ void opt_update_d(const OptParamsD& o, float g, float& w, float& s1, float& s2) {
    if (o.kind == WD_OPT_ADAGRAD) {
        s1 += g * g;
        w -= o.lr * g / sqrtf(s1);
    } else if (o.kind == WD_OPT_FTRL) {
        float n1 = s1 + g * g;
        float z1 = s2 + g - (sqrtf(n1) - sqrtf(s1)) / o.lr * w;
        float wn = 0.f;
        if (fabsf(z1) > o.l1) wn = (copysignf(o.l1, z1) - z1) / (sqrtf(n1) / o.lr + 2.f * o.l2);
        w = wn; s1 = n1; s2 = z1;
    } else if (o.kind == WD_OPT_ADAM) {             // ApplyAdam; bpow = {beta1^t, beta2^t} (device: advances after every step)
        const float lr_t = o.lr * sqrtf(1.f - o.bpow[1]) / (1.f - o.bpow[0]);
        s1 += (g - s1) * (1.f - o.beta1);
        s2 += (g * g - s2) * (1.f - o.beta2);
        w -= lr_t * s1 / (sqrtf(s2) + o.epsilon);
    } else if (o.kind == WD_OPT_RMSPROP) {          // ApplyRMSProp (not centered)
        s1 += (g * g - s1) * (1.f - o.rho);
        s2 = s2 * o.momentum + (g * o.lr) / sqrtf(s1 + o.epsilon);
        w -= s2;
    } else {
        w -= o.lr * g;
    }
}
// tf32 hi/lo split of a weight for the 3xTF32 engine (same split the GEMM applies to activations in shared memory), stored at
// e in W [K, N] and at et in Wt [N, K]
__device__ __forceinline__ void store_split(float* __restrict__ W_hi, float* __restrict__ W_lo, float* __restrict__ Wt_hi,
                                            float* __restrict__ Wt_lo, int64_t e, int64_t et, float w) {
    float hi = __uint_as_float(__float_as_uint(w) & 0xFFFFE000u), lo = w - hi;
    W_hi[e] = hi;
    W_lo[e] = lo;
    Wt_hi[et] = hi;
    Wt_lo[et] = lo;
}
// applies the optimizer over the dense arena (fp32 operand family); kernels also refresh their transposed copy Wt[n][k] and the
// tf32 hi / lo splits
__global__ void dense_apply_kernel(const DenseTensor* __restrict__ T, int nt, int64_t total, const float* __restrict__ G,
                                   float* __restrict__ P, float* __restrict__ S1, float* __restrict__ S2, float* __restrict__ Wt,
                                   float* __restrict__ W_hi, float* __restrict__ W_lo, float* __restrict__ Wt_hi, float* __restrict__ Wt_lo,
                                   OptParamsD dnn, OptParamsD lin, int lin_tensor) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int lo = 0, hi = nt - 1;
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            if (T[mid].off <= i) lo = mid; else hi = mid - 1;
        }
        const DenseTensor t = T[lo];
        if (i - t.off >= t.count) continue;
        float w = P[i], s1 = S1[i], s2 = S2[i];
        opt_update_d(lo == lin_tensor ? lin : dnn, G[i], w, s1, s2);
        P[i] = w; S1[i] = s1; S2[i] = s2;
        if (t.wt_off >= 0) {
            int64_t e = i - t.off;
            int k = (int)(e / t.cols), n = (int)(e % t.cols);
            Wt[t.wt_off + (int64_t)n * t.rows + k] = w;
            store_split(W_hi, W_lo, Wt_hi, Wt_lo, t.wt_off + e, t.wt_off + (int64_t)n * t.rows + k, w);
        }
    }
}
// Vectorised dense-gradient reduction / optimizer for the bf16 operand family (no transposed weight copies to scatter): one thread per
// four consecutive arena floats (tensor offsets, partial strides and kernel widths are multiples of 4), one tensor lookup per
// thread instead of per element.
//   MODE 0: G = sum of the live partials                      (data-parallel runs: G is exchanged before the optimizer)
//   MODE 1: optimizer from G                                   (after the exchange)
//   MODE 2: both in one pass, G never materialised            (single-GPU step: saves a 6 MB round trip and a launch)
template <int MODE>
__global__ void __launch_bounds__(256) dense_vec_kernel(const DenseTensor* __restrict__ T, int nt, int64_t total4, const float* __restrict__ gpart,
                                                        float* __restrict__ G, float* __restrict__ P, float* __restrict__ S1, float* __restrict__ S2,
                                                        __nv_bfloat16* __restrict__ Wq_hi, __nv_bfloat16* __restrict__ Wq_lo, OptParamsD dnn, OptParamsD lin, int lin_tensor,
                                                        int live_row_tiles, int64_t begin4, int64_t hole_lo4, int64_t hole_hi4) {
    // arena range [begin4, total4) minus the hole [hole_lo4, hole_hi4): the single-GPU step updates everything but the first
    // layer's kernel on a side stream while that kernel's weight gradient is still being computed (dense_apply_split)
    for (int64_t i4 = begin4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i4 < total4; i4 += (int64_t)gridDim.x * blockDim.x) {
        if (i4 >= hole_lo4 && i4 < hole_hi4) continue;
        const int64_t i = i4 * 4;
        int lo = 0, hi = nt - 1;
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            if (T[mid].off <= i) lo = mid; else hi = mid - 1;
        }
        const DenseTensor t = T[lo];
        const int64_t e = i - t.off;
        if (e >= t.count) {                                               // alignment gap between tensors
            if (MODE == 0) reinterpret_cast<float4*>(G)[i4] = make_float4(0.f, 0.f, 0.f, 0.f);
            continue;
        }
        float4 g;
        if (MODE != 1) {
            const int parts = t.g_rowtiles ? live_row_tiles : t.gparts;
            const float* p = gpart + t.gpart_off + e;
            g = make_float4(0.f, 0.f, 0.f, 0.f);
            int q = 0;
            for (; q + 4 <= parts; q += 4) {                              // four partials in flight, summed in index order
                const float4 v0 = *reinterpret_cast<const float4*>(p + (int64_t)q * t.gstride);
                const float4 v1 = *reinterpret_cast<const float4*>(p + (int64_t)(q + 1) * t.gstride);
                const float4 v2 = *reinterpret_cast<const float4*>(p + (int64_t)(q + 2) * t.gstride);
                const float4 v3 = *reinterpret_cast<const float4*>(p + (int64_t)(q + 3) * t.gstride);
                g.x += v0.x; g.y += v0.y; g.z += v0.z; g.w += v0.w;
                g.x += v1.x; g.y += v1.y; g.z += v1.z; g.w += v1.w;
                g.x += v2.x; g.y += v2.y; g.z += v2.z; g.w += v2.w;
                g.x += v3.x; g.y += v3.y; g.z += v3.z; g.w += v3.w;
            }
            for (; q < parts; ++q) {
                const float4 v = *reinterpret_cast<const float4*>(p + (int64_t)q * t.gstride);
                g.x += v.x; g.y += v.y; g.z += v.z; g.w += v.w;
            }
            if (e + 1 >= t.count) g.y = 0.f;                              // tensors shorter than the vector (scalar biases): the tail
            if (e + 2 >= t.count) g.z = 0.f;                              // lanes read neighbouring partials, not gradients
            if (e + 3 >= t.count) g.w = 0.f;
            if (MODE == 0) { reinterpret_cast<float4*>(G)[i4] = g; continue; }
        } else {
            g = reinterpret_cast<const float4*>(G)[i4];
        }
        const OptParamsD o = lo == lin_tensor ? lin : dnn;
        float4 w = reinterpret_cast<float4*>(P)[i4], s1 = reinterpret_cast<float4*>(S1)[i4], s2 = reinterpret_cast<float4*>(S2)[i4];
        opt_update_d(o, g.x, w.x, s1.x, s2.x);
        if (e + 1 < t.count) opt_update_d(o, g.y, w.y, s1.y, s2.y);
        if (e + 2 < t.count) opt_update_d(o, g.z, w.z, s1.z, s2.z);
        if (e + 3 < t.count) opt_update_d(o, g.w, w.w, s1.w, s2.w);
        reinterpret_cast<float4*>(P)[i4] = w;
        reinterpret_cast<float4*>(S1)[i4] = s1;
        reinterpret_cast<float4*>(S2)[i4] = s2;
        if (t.wt_off >= 0)                                                // bf16 hi / lo copies of W [K, N] (what the GEMMs read)
            store_split4(Wq_hi + t.wt_off + e, Wq_lo + t.wt_off + e, w.x, w.y, w.z, w.w);
    }
}

// Rewrites the GEMM operand copies of the weights from P (after init / tensor upload): Wt and the tf32 splits for the fp32
// family, the bf16 splits (Wq_hi non-null) for the bf16 family
__global__ void weight_copies_kernel(const DenseTensor* __restrict__ T, int nt, int64_t total, const float* __restrict__ P, float* __restrict__ Wt,
                                     float* __restrict__ W_hi, float* __restrict__ W_lo, float* __restrict__ Wt_hi, float* __restrict__ Wt_lo,
                                     __nv_bfloat16* __restrict__ Wq_hi, __nv_bfloat16* __restrict__ Wq_lo) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int lo = 0, hi = nt - 1;
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            if (T[mid].off <= i) lo = mid; else hi = mid - 1;
        }
        const DenseTensor t = T[lo];
        if (t.wt_off >= 0 && i - t.off < t.count) {
            int64_t e = i - t.off;
            if (Wq_hi) {
                __nv_bfloat16 qh, ql;
                split_bf16(P[i], qh, ql);
                Wq_hi[t.wt_off + e] = qh;
                Wq_lo[t.wt_off + e] = ql;
                continue;
            }
            int k = (int)(e / t.cols), n = (int)(e % t.cols);
            Wt[t.wt_off + (int64_t)n * t.rows + k] = P[i];
            store_split(W_hi, W_lo, Wt_hi, Wt_lo, t.wt_off + e, t.wt_off + (int64_t)n * t.rows + k, P[i]);
        }
    }
}
int refresh_weight_copies(WdModel* m) {
    if (m->dense_count == 0) return WD_OK;
    weight_copies_kernel<<<grid_for(m->dense_count, 256), 256, 0, m->stream>>>(m->d_dense_desc, (int)m->dense.size(), m->dense_count, m->d_P, m->d_Wt,
                                                                               m->d_W_hi, m->d_W_lo, m->d_Wt_hi, m->d_Wt_lo, m->d_Wq_hi, m->d_Wq_lo);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ------------------------------------------------------------------------------------------ host drivers
// a layer input: src -1 is the deep input X0, src >= 0 hidden layer src of the same tower
static const float* src_ptr(WdModel* m, Tower& tw, int src) { return src < 0 ? m->d_X0 : tw.layers[src].H; }
static const __nv_bfloat16* src_split(WdModel* m, Tower& tw, int src, int part) { return src < 0 ? m->d_X0s[part] : tw.layers[src].Hs[part]; }
static int src_ld(WdModel* m, Tower& tw, int src) { return src < 0 ? m->d0_phys : tw.layers[src].N_phys; }

// ---- GEMM operands of a hidden layer (A, B zero-initialised), read off the operand-family table at the top of this file.
// GemmB = {ptr, ld, tf32_hi, tf32_lo, hi, lo}.
// forward: A = the layer's input segments, B = its kernel
static void fwd_operands(WdModel* m, Tower& tw, const Layer& L, GemmA& A, GemmB& B) {
    const int64_t wo = m->dense[L.t_kernel].wt_off;
    A.n = L.n_in_segs;
    for (int s = 0; s < L.n_in_segs; ++s) {
        const int src = L.segs[s].src;
        A.ld[s] = src_ld(m, tw, src); A.k[s] = L.segs[s].width_phys;
        if (m->operands == kFp32Operands) A.ptr[s] = src_ptr(m, tw, src);
        else { A.hi[s] = src_split(m, tw, src, 0); A.lo[s] = src_split(m, tw, src, 1); }
    }
    if (m->operands == kFp32Operands) B = GemmB{m->d_Wt + wo, L.K_phys, m->d_Wt_hi + wo, m->d_Wt_lo + wo, nullptr, nullptr};
    else B = GemmB{nullptr, L.N_phys, nullptr, nullptr, m->d_Wq_hi + wo, m->d_Wq_lo + wo};
}
// data gradient into input segment sg: A = the layer's dZ, B = the kernel rows that segment feeds
static void dgrad_operands(WdModel* m, const Layer& L, const Seg& sg, GemmA& A, GemmB& B) {
    const DenseTensor& tk = m->dense[L.t_kernel];
    const int64_t eo = (int64_t)sg.k_off * L.N_phys, wo = tk.wt_off + eo;
    A.n = 1; A.ld[0] = L.N_phys; A.k[0] = L.N_phys;
    if (m->operands == kFp32Operands) {
        A.ptr[0] = L.dZ;
        B = GemmB{m->d_P + tk.off + eo, L.N_phys, m->d_W_hi + wo, m->d_W_lo + wo, nullptr, nullptr};
    } else {
        A.hi[0] = L.dZs[0]; A.lo[0] = L.dZs[1];
        B = GemmB{nullptr, L.N_phys, nullptr, nullptr, m->d_Wq_hi + wo, m->d_Wq_lo + wo};
    }
}
// weight gradient of the kernel rows input segment sg feeds: A = that input, B = the layer's dZ, the batch being the reduction
static void wgrad_operands(WdModel* m, Tower& tw, const Layer& L, const Seg& sg, GemmA& A, GemmB& B) {
    A.n = 1;
    if (m->operands == kFp32Operands) {                // transposed copies; the batch padded to 16 (rows past it are zero)
        A.ptr[0] = sg.src < 0 ? m->d_X0T : tw.layers[sg.src].HT; A.ld[0] = m->ldt; A.k[0] = (m->dbatch.B + 15) / 16 * 16;
        B = GemmB{L.dZT, m->ldt, nullptr, nullptr, nullptr, nullptr};
    } else {                                           // row-major [B, width] copies (TMA zero-fills the batch tail)
        A.hi[0] = src_split(m, tw, sg.src, 0); A.lo[0] = src_split(m, tw, sg.src, 1); A.ld[0] = src_ld(m, tw, sg.src); A.k[0] = m->dbatch.B;
        B = GemmB{nullptr, L.N_phys, nullptr, nullptr, L.dZs[0], L.dZs[1]};
    }
}

int mlp_forward(WdModel* m, bool train) {
    const int B = m->dbatch.B;
    if (!m->use_deep) return WD_OK;
    if (m->operands == kBf16Operands) {                // bf16 hi / lo copies of X0
        const int64_t n4 = (int64_t)B * m->d0_phys / 4;
        x0_split_kernel<<<grid_for(n4, 256), 256, 0, m->stream>>>(m->d_X0, n4, m->d_X0s[0], m->d_X0s[1]);
        m->launches++;
    } else if (train) {                                // X0T for the first layer's weight gradient
        int Bp = (B + 127) / 128 * 128;
        dim3 g((m->d0_phys + 31) / 32, (Bp + 31) / 32);
        transpose_kernel<<<g, dim3(32, 8), 0, m->stream>>>(m->d_X0, m->d0_phys, B, Bp, m->d0_phys, m->d_X0T, m->ldt);
        m->launches++;
    }
    for (auto& tw : m->towers) {
        for (int l = 0; l < tw.n_hidden; ++l) {
            Layer& L = tw.layers[l];
            m->cur_layer = l;
            GemmA A{}; GemmB W{};
            fwd_operands(m, tw, L, A, W);
            // the layer's outputs: whichever of H, HT (train steps) and the bf16 copies Hs the model has
            Epi ep{};
            ep.A_out = L.A; ep.H_out = L.H; ep.ldh = L.N_phys;
            ep.HT = train ? L.HT : nullptr; ep.ldt = m->ldt;
            ep.Hs_hi = L.Hs[0]; ep.Hs_lo = L.Hs[1];
            ep.bias = m->d_P + m->dense[L.t_bias].off;
            ep.gamma = L.t_gamma >= 0 ? m->d_P + m->dense[L.t_gamma].off : nullptr;
            ep.beta = L.t_beta >= 0 ? m->d_P + m->dense[L.t_beta].off : nullptr;
            ep.n_logical = L.N; ep.act = m->activation; ep.bn = m->batch_norm; ep.m_valid = B;
            int rc = run_gemm(m, EPI_FWD, A, W, B, L.N_phys, ep);
            if (rc) return rc;
            if (train && m->dropout_rate > 0.f) {              // tf.layers.dropout(training=True): TRAIN steps only (dnn.py:111-112)
                const DropArgs dr{m->dropout_rate, m->dropout_seed, m->d_step, (int)(&tw - &m->towers[0]) * 64 + l, drop_row0(m)};
                dropout_fwd_kernel<<<grid_for((int64_t)B * L.N_phys, 256), 256, 0, m->stream>>>(B, L.N_phys, L.N, L.A, L.N_phys, ep.gamma, ep.beta, m->batch_norm,
                    L.H, L.Hs[0], L.Hs[1], ep.HT, m->ldt, dr);
                m->launches++;
            }
        }
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

int loss_forward(WdModel* m, bool need_grad) {
    const int B = m->dbatch.B;
    const int ntow = m->use_deep ? (int)m->towers.size() : 0;      // <= kMaxTowers (wd_model_create)
    HeadIn in{};
    in.n = ntow;
    for (int t = 0; t < ntow; ++t) {
        Tower& tw = m->towers[t];
        Layer& LL = tw.layers[tw.n_hidden];
        in.S[t].n = LL.n_in_segs;
        for (int s = 0; s < LL.n_in_segs; ++s) {
            in.S[t].ptr[s] = src_ptr(m, tw, LL.segs[s].src);
            in.S[t].ld[s] = src_ld(m, tw, LL.segs[s].src);
            in.S[t].k[s] = LL.segs[s].width_phys;
            in.S[t].koff[s] = LL.segs[s].k_off;
        }
        in.kernel[t] = m->d_P + m->dense[LL.t_kernel].off;
        in.bias[t] = m->d_P + m->dense[LL.t_bias].off;
        in.tower_logit[t] = tw.logit;
    }
    const int blocks = grid_for((int64_t)B * 8, 256, 512);               // eight lanes per example (loss_part holds 512 block partials)
    logits_head_kernel<<<blocks, 256, 0, m->stream>>>(in, B, m->use_wide ? m->d_wide_logit : nullptr, m->dbatch.label,
                                                     m->dbatch.weight, m->d_logits, need_grad ? m->d_dlogit : nullptr, m->d_loss_part,
                                                     m->d_head_counter, m->d_loss);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

int mlp_backward(WdModel* m) {
    const int B = m->dbatch.B;
    if (!m->use_deep) return WD_OK;
    const int rts = (B + 127) / 128;
    const int Bk = (B + 15) / 16 * 16;                                // reduction length of wgrad
    bool dx0_written = false;
    const bool need_dx0 = !m->tables.empty();
    const bool bf16_ops = m->operands == kBf16Operands;
    for (auto& tw : m->towers) {
        std::vector<char> written(tw.n_hidden, 0);
        std::vector<int> readers(tw.n_hidden, 0);
        std::vector<char> fused(tw.n_hidden, 0);
        for (int l = 0; l <= tw.n_hidden; ++l)
            for (int s = 0; s < tw.layers[l].n_in_segs; ++s)
                if (tw.layers[l].segs[s].src >= 0) readers[tw.layers[l].segs[s].src] += (l == tw.n_hidden ? 2 : 1);   // the logits layer's kernel is not a GEMM
        auto grad_dst = [&](int src, float** p, int* ld, int* acc) {
            if (src < 0) { *p = m->d_dX0; *ld = m->d0_phys; *acc = dx0_written ? 1 : 0; dx0_written = true; }
            else { *p = tw.layers[src].dH; *ld = tw.layers[src].N_phys; *acc = written[src] ? 1 : 0; written[src] = 1; }
        };
        // ---- logits layer
        Layer& LL = tw.layers[tw.n_hidden];
        const DenseTensor& tk = m->dense[LL.t_kernel];
        const DenseTensor& tb = m->dense[LL.t_bias];
        for (int s = 0; s < LL.n_in_segs; ++s) {
            const Seg& sg = LL.segs[s];
            const float* src = src_ptr(m, tw, sg.src);
            int ld = src_ld(m, tw, sg.src);
            dim3 g((sg.width_phys + 63) / 64, rts);
            float* dst = nullptr; int dld = 0, acc = 0;
            if (!(sg.src < 0 && !need_dx0)) grad_dst(sg.src, &dst, &dld, &acc);
            // (the first segment of the first tower also leaves the wide bias's gradient partials: both are tile sums of dlogit)
            const bool wb = m->use_wide && s == 0 && &tw == &m->towers.front();
            // bf16 family, a hidden layer read by the logits layer alone: its activation / batch-norm backward runs in the same
            // pass (logits_act_bwd_q_kernel), so its dH is never stored and act_bn_bwd_q_kernel is not launched for it
            if (bf16_ops && LL.n_in_segs == 1 && sg.src >= 0 && readers[sg.src] == 2 && m->dropout_rate <= 0.f &&
                sg.width_phys == tw.layers[sg.src].N_phys) {
                Layer& S = tw.layers[sg.src];
                logits_act_bwd_q_kernel<<<dim3((S.N_phys + 63) / 64, rts), 256, 0, m->stream>>>(B, S.N_phys, S.N, src, ld, S.A, S.N_phys, m->d_dlogit,
                    m->d_P + tk.off + sg.k_off, S.t_gamma >= 0 ? m->d_P + m->dense[S.t_gamma].off : nullptr, m->activation, m->batch_norm,
                    m->d_gpart + tk.gpart_off + sg.k_off, tk.gstride, m->d_gpart + tb.gpart_off, tb.gstride,
                    wb ? m->d_gpart + m->dense[0].gpart_off : nullptr, wb ? m->dense[0].gstride : 0,
                    m->d_gpart + m->dense[S.t_bias].gpart_off, S.t_gamma >= 0 ? m->d_gpart + m->dense[S.t_gamma].gpart_off : nullptr,
                    S.t_beta >= 0 ? m->d_gpart + m->dense[S.t_beta].gpart_off : nullptr, m->dense[S.t_bias].gstride, S.dZs[0], S.dZs[1]);
                m->launches++;
                fused[sg.src] = 1;
                continue;
            }
            logits_bwd_kernel<<<g, 256, 0, m->stream>>>(B, sg.width_phys, src, ld, m->d_dlogit, m->d_P + tk.off + sg.k_off,
                                                       m->d_gpart + tk.gpart_off + sg.k_off, tk.gstride,
                                                       s == 0 ? m->d_gpart + tb.gpart_off : nullptr, tb.gstride,
                                                       wb ? m->d_gpart + m->dense[0].gpart_off : nullptr, wb ? m->dense[0].gstride : 0, dst, dld, acc);
            m->launches++;
        }
        // ---- hidden layers, last to first
        for (int l = tw.n_hidden - 1; l >= 0; --l) {
            Layer& L = tw.layers[l];
            m->cur_layer = l;
            float* pb = m->d_gpart + m->dense[L.t_bias].gpart_off;
            float* pg = L.t_gamma >= 0 ? m->d_gpart + m->dense[L.t_gamma].gpart_off : nullptr;
            float* pbe = L.t_beta >= 0 ? m->d_gpart + m->dense[L.t_beta].gpart_off : nullptr;
            if (!written[l] && !fused[l]) {                           // layer output unused downstream (cannot happen for valid modes)
                WD_CUDA(cudaMemsetAsync(L.dH, 0, (size_t)m->max_batch_pad * L.N_phys * sizeof(float), m->stream));
            }
            dim3 g((L.N_phys + 31) / 32, rts);
            const DropArgs dr{m->dropout_rate, m->dropout_seed, m->d_step, (int)(&tw - &m->towers[0]) * 64 + l, drop_row0(m)};
            if (fused[l]) {
                // dZ and the partials of this layer were written by logits_act_bwd_q_kernel
            } else if (bf16_ops)
                act_bn_bwd_q_kernel<<<dim3((L.N_phys + 63) / 64, rts), 256, 0, m->stream>>>(B, L.N_phys, L.N, L.dH, L.A, L.N_phys,
                    L.t_gamma >= 0 ? m->d_P + m->dense[L.t_gamma].off : nullptr, m->activation, m->batch_norm, pb, pg, pbe,
                    m->dense[L.t_bias].gstride, L.dZs[0], L.dZs[1], dr);
            else
            act_bn_bwd_kernel<<<g, 256, 0, m->stream>>>(B, L.N_phys, L.N, L.dH, L.A, L.N_phys,
                                                       L.t_gamma >= 0 ? m->d_P + m->dense[L.t_gamma].off : nullptr, m->activation,
                                                       m->batch_norm, L.dZ, L.dZT, m->ldt, pb, pg, pbe, m->dense[L.t_bias].gstride, dr);
            if (!fused[l]) m->launches++;
            // data gradients first: the deep-input gradient dX0 is what the embedding backward waits for, so it is
            // produced before this layer's weight gradients (which then overlap the sparse backward on the side stream)
            for (int s = 0; s < L.n_in_segs; ++s) {
                const Seg& sg = L.segs[s];
                if (sg.src < 0 && !need_dx0) continue;
                float* dst; int dld, acc;
                grad_dst(sg.src, &dst, &dld, &acc);
                GemmA A{}; GemmB W{};
                dgrad_operands(m, L, sg, A, W);
                Epi ep{};
                ep.C = dst; ep.ldc = dld; ep.accumulate = acc;
                int rc = run_gemm(m, EPI_STORE, A, W, B, sg.width_phys, ep);
                if (rc) return rc;
            }
            if (l == 0 && &tw == &m->towers.back() && need_dx0 && m->ev_dx0 && m->record_dx0) {
                WD_CUDA(cudaEventRecord(m->ev_dx0, m->stream));        // dX0 is complete from here on
                m->dx0_recorded = true;
            }
        }
        // ---- weight gradients, after EVERY data gradient of the tower: dX0 exists as early as the dependency chain allows, and
        // the embedding backward on its side stream (sums + row updates, the longest tail of the step) runs under all of the
        // tower's weight-gradient GEMMs and the dense optimizer instead of under the last one only
        for (int l = tw.n_hidden - 1; l >= 0; --l) {
            Layer& L = tw.layers[l];
            m->cur_layer = l;
            const DenseTensor& tkn = m->dense[L.t_kernel];
            if (l == 0 && m->record_wgrad_rest && m->towers.size() == 1 && L.n_in_segs == 1) {
                // every gradient partial except the first layer's kernel is final from here on
                WD_CUDA(cudaEventRecord(m->ev_wgrad_rest, m->stream));
                m->dense_split_tensor = L.t_kernel;
            }
            for (int s = 0; s < L.n_in_segs; ++s) {
                const Seg& sg = L.segs[s];
                // weight gradient of the rows fed by this segment: [width_phys, N], split over the batch
                GemmA A{}; GemmB W{};
                wgrad_operands(m, tw, L, sg, A, W);
                Epi ep{};
                ep.C = m->d_gpart + tkn.gpart_off + (int64_t)sg.k_off * L.N_phys; ep.ldc = L.N_phys; ep.split_stride = tkn.gstride;
                const int ks = ((Bk + L.wgrad_splits - 1) / L.wgrad_splits + 31) / 32 * 32;     // (engines round it up to their k-block)
                int rc = run_gemm(m, EPI_WGRAD, A, W, sg.width_phys, L.N_phys, ep, L.wgrad_splits, ks);
                if (rc) return rc;
            }
        }
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ---- crelu layers (reference python/lib/utils/model_util.py:45-50, tf.nn.crelu): built as relu layers of twice the width whose
// kernel / bias columns n + u hold minus columns n.  The backward leaves gradients for both halves; the variable's gradient is their
// difference (d/dW of [xW | -xW]).  crelu_fold puts it into the first half of every live partial and zeroes the second half, so the
// reduction, the exchange and the optimizer kernels see a plain tensor; crelu_mirror re-derives the tied half (parameter negated,
// optimizer slots copied) and refreshes the GEMM operand copies after the optimizer.
__global__ void crelu_fold_kernel(float* __restrict__ gp, int parts, int64_t gstride, int rows, int cols, int u) {
    const int64_t total = (int64_t)parts * rows * u;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int n = (int)(i % u);
        const int64_t pr = i / u;
        float* q = gp + (pr / rows) * gstride + (pr % rows) * cols + n;
        q[0] -= q[u];
        q[u] = 0.f;
    }
}
__global__ void crelu_mirror_kernel(float* __restrict__ P, float* __restrict__ S1, float* __restrict__ S2, int rows, int cols, int u) {
    const int64_t total = (int64_t)rows * u;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = (i / u) * cols + i % u;
        P[e + u] = -P[e];
        S1[e + u] = S1[e];
        S2[e + u] = S2[e];
    }
}
static int crelu_fold(WdModel* m) {
    const int rts = (m->dbatch.B + 127) / 128;
    for (const DenseTensor& t : m->dense) {
        if (!t.mirror_u) continue;
        const int parts = t.g_rowtiles ? rts : t.gparts;
        crelu_fold_kernel<<<grid_for((int64_t)parts * t.rows * t.mirror_u, 256), 256, 0, m->stream>>>(m->d_gpart + t.gpart_off, parts, t.gstride, t.rows, t.cols,
                                                                                                    t.mirror_u);
        m->launches++;
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
static int crelu_mirror(WdModel* m) {
    for (const DenseTensor& t : m->dense) {
        if (!t.mirror_u) continue;
        crelu_mirror_kernel<<<grid_for((int64_t)t.rows * t.mirror_u, 256), 256, 0, m->stream>>>(m->d_P + t.off, m->d_S1 + t.off, m->d_S2 + t.off, t.rows, t.cols,
                                                                                              t.mirror_u);
        m->launches++;
    }
    WD_CUDA(cudaGetLastError());
    return refresh_weight_copies(m);
}

int dense_reduce_grads(WdModel* m) {
    if (m->dense_count == 0) return WD_OK;
    const int rts = (m->dbatch.B + 127) / 128;
    if (m->crelu) { int rc = crelu_fold(m); if (rc) return rc; }
    if (m->operands == kBf16Operands) {
        if (m->fuse_dense) return WD_OK;                              // single-GPU step: reduced inside dense_apply's kernel
        OptParamsD z{};
        dense_vec_kernel<0><<<grid_for(m->dense_count / 4, 256), 256, 0, m->stream>>>(m->d_dense_desc, (int)m->dense.size(), m->dense_count / 4, m->d_gpart,
            m->d_G, nullptr, nullptr, nullptr, nullptr, nullptr, z, z, -1, rts, 0, 0, 0);
        m->launches++;
        WD_CUDA(cudaGetLastError());
        return WD_OK;
    }
    dense_reduce_kernel<<<grid_for(m->dense_count, 256), 256, 0, m->stream>>>(m->d_dense_desc, (int)m->dense.size(), m->dense_count,
                                                                             m->d_gpart, m->d_G, rts);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

static int dense_apply_plain(WdModel* m) {
    if (m->dense_count == 0) return WD_OK;
    OptParamsD d = make_opt_d(m->dnn_opt, m->d_bpow + 2);
    OptParamsD l = make_opt_d(m->lin_opt, m->d_bpow);
    int lin_tensor = m->use_wide ? 0 : -1;                       // tensor 0 is the wide bias when the wide part exists
    if (m->operands == kBf16Operands) {
        const int rts = (m->dbatch.B + 127) / 128;
        const int g = grid_for(m->dense_count / 4, 256);
        if (m->fuse_dense) {
            // part: 0 = whole arena, 1 = only the first layer's kernel (the rest was updated on a side stream), 2 = all but that kernel
            int64_t b4 = 0, e4 = m->dense_count / 4, hlo = 0, hhi = 0;
            if (m->dense_part && m->dense_split_tensor >= 0) {
                const DenseTensor& t = m->dense[m->dense_split_tensor];
                const int64_t k0 = t.off / 4, k1 = (t.off + t.count + 3) / 4;
                if (m->dense_part == 1) { b4 = k0; e4 = k1; } else { hlo = k0; hhi = k1; }
            }
            dense_vec_kernel<2><<<grid_for(e4 - b4, 256), 256, 0, m->stream>>>(m->d_dense_desc, (int)m->dense.size(), e4, m->d_gpart, m->d_G, m->d_P,
                                                                                m->d_S1, m->d_S2, m->d_Wq_hi, m->d_Wq_lo, d, l, lin_tensor, rts, b4, hlo, hhi);
        } else
            dense_vec_kernel<1><<<g, 256, 0, m->stream>>>(m->d_dense_desc, (int)m->dense.size(), m->dense_count / 4, m->d_gpart, m->d_G, m->d_P, m->d_S1,
                                                          m->d_S2, m->d_Wq_hi, m->d_Wq_lo, d, l, lin_tensor, rts, 0, 0, 0);
        m->launches++;
        WD_CUDA(cudaGetLastError());
        return WD_OK;
    }
    dense_apply_kernel<<<grid_for(m->dense_count, 256), 256, 0, m->stream>>>(m->d_dense_desc, (int)m->dense.size(), m->dense_count, m->d_G,
                                                                            m->d_P, m->d_S1, m->d_S2, m->d_Wt, m->d_W_hi, m->d_W_lo, m->d_Wt_hi,
                                                                            m->d_Wt_lo, d, l, lin_tensor);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// optimizer of the dense arena (+ the tied halves of crelu layers)
int dense_apply(WdModel* m) {
    int rc = dense_apply_plain(m);
    if (!rc && m->crelu && m->dense_count > 0) rc = crelu_mirror(m);
    return rc;
}

}  // namespace wd
