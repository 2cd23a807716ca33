// Shared GEMM interface of the MLP engines (FFMA in mlp.cu, wgmma in gemm_tc.cu and gemm_bf16.cu): operand descriptions,
// epilogue description and the activation functions (reference python/lib/utils/model_util.py:28-59).  Which stored copy each
// operand is read from is tabled at the top of mlp.cu.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"

namespace wd {

// --------------------------------------------------------------------------------------------- activations
__device__ __forceinline__ float act_fwd(int kind, float z) {
    switch (kind) {
        case WD_ACT_RELU: return fmaxf(z, 0.f);
        case WD_ACT_RELU6: return fminf(fmaxf(z, 0.f), 6.f);
        case WD_ACT_SIGMOID: return 1.f / (1.f + expf(-z));
        case WD_ACT_TANH: return tanhf(z);
        case WD_ACT_LEAKY_RELU: return z > 0.f ? z : 0.2f * z;
        case WD_ACT_ELU: return z > 0.f ? z : expm1f(z);
        case WD_ACT_SELU: return 1.0507009873554805f * (z > 0.f ? z : 1.6732632423543772f * expm1f(z));
        case WD_ACT_SOFTPLUS: return fmaxf(z, 0.f) + log1pf(expf(-fabsf(z)));
        case WD_ACT_SOFTSIGN: return z / (1.f + fabsf(z));
    }
    return z;
}
// derivative expressed through the stored post-activation value a
__device__ __forceinline__ float act_bwd(int kind, float a) {
    switch (kind) {
        case WD_ACT_RELU: return a > 0.f ? 1.f : 0.f;
        case WD_ACT_RELU6: return (a > 0.f && a < 6.f) ? 1.f : 0.f;
        case WD_ACT_SIGMOID: return a * (1.f - a);
        case WD_ACT_TANH: return 1.f - a * a;
        case WD_ACT_LEAKY_RELU: return a > 0.f ? 1.f : 0.2f;
        case WD_ACT_ELU: return a > 0.f ? 1.f : a + 1.f;
        case WD_ACT_SELU: return a > 0.f ? 1.0507009873554805f : a + 1.0507009873554805f * 1.6732632423543772f;
        case WD_ACT_SOFTPLUS: return 1.f - expf(-a);
        case WD_ACT_SOFTSIGN: { float t = 1.f - fabsf(a); return t * t; }
    }
    return 1.f;
}

// ------------------------------------------------------------------------------------------- FFMA GEMM
struct GemmA {                         // A operand: up to kMaxSegs K-contiguous segments
    int n;
    const float* ptr[kMaxSegs];
    int ld[kMaxSegs];
    int k[kMaxSegs];                   // multiple of 16
    const __nv_bfloat16* hi[kMaxSegs]; // 3xBF16 engine: the same segments pre-split into bf16 hi / lo copies (same ld)
    const __nv_bfloat16* lo[kMaxSegs];
};
struct GemmB {                         // B operand: one segment (host side only; the FFMA kernel takes ptr / ld)
    const float* ptr; int ld;
    const float *tf32_hi, *tf32_lo;    // 3xTF32 forward / data gradient: ptr pre-split into tf32 hi / lo copies (same ld)
    const __nv_bfloat16 *hi, *lo;      // 3xBF16 engine: bf16 hi / lo copies (same ld)
};
enum { EPI_FWD = 0, EPI_STORE = 1, EPI_WGRAD = 2 };
struct Epi {
    float* C; int ldc;                 // STORE / WGRAD target
    int accumulate;                    // STORE: C += acc
    float* A_out; float* H_out; int ldh;   // FWD outputs
    float* HT; int ldt;                // FWD transposed output (nullable)
    const float *bias, *gamma, *beta;
    int n_logical, act, bn;
    int m_valid;                       // rows >= m_valid are written as zero (transposed padding)
    int64_t split_stride;              // WGRAD: floats between split partials
    // 3xBF16 engine, FWD: the layer output leaves as bf16 hi / lo copies, row-major [M, ldh] (H_out may then be NULL)
    __nv_bfloat16 *Hs_hi, *Hs_lo;
    // Nothing reads these 40 bytes.  They keep the parameter block of the wgmma GEMM kernels at the layout those were tuned with:
    // without them ptxas schedules the forward GEMMs of both engines differently, and those ran 11 % slower (H100 80GB HBM3, 700 W,
    // Criteo shape: 8.47 M against 8.84 M examples/s for the whole step).
    uint64_t reserved[5];
};

// wgmma engines; tc_gemm returns WD_EUNSUPPORTED when the shape is not covered
int tc_gemm(WdModel* m, int mode, const GemmA& A, const GemmB& B, int M, int N, const Epi& ep, int splits, int ksplit_len);
int tc_gemm_bf16(WdModel* m, int mode, const GemmA& A, const GemmB& B, int M, int N, const Epi& ep, int splits, int ksplit_len);
// 2-D TMA tensor map of a row-major fp32 or bf16 matrix [rows, cols] with leading dimension ld (elements): box = one 128-byte
// row of columns x box_rows, 128-byte swizzle.  Encoded maps are cached (gemm_tc.cu).
int make_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, const void* ptr, int rows, int cols, int ld, int box_rows);

// ---- dropout (tf.layers.dropout after a hidden layer's activation, TRAIN only; reference dnn.py:111-112).  TensorFlow's random
// stream cannot be reproduced, so the keep mask is DEFINED by a counter-based generator shared bit for bit with the oracle
// (oracle/model.py drop_keep): element (m, n) of layer `layer_id` in train step `step` is kept iff
//   u >= rate,  u = top 24 bits of splitmix64(key ^ (m * 65536 + n)) / 2^24,  key = splitmix64(seed ^ step * GOLDEN ^ layer_id << 48)
// and kept elements are scaled by 1 / (1 - rate).  Nothing is stored: the backward regenerates the mask.
// m is the row of the global batch: row0 + the local row, row0 = rank * max_batch on a row-sharded rank (drop_row0) and 0 on one
// GPU.  So no two ranks share a mask, and G ranks with full batches draw the mask one GPU draws on their concatenated batch.
struct DropArgs { float rate; unsigned long long seed; const unsigned int* step; int layer_id; unsigned int row0; };
__device__ __forceinline__ unsigned long long splitmix64_dev(unsigned long long x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}
__device__ __forceinline__ unsigned long long drop_key(const DropArgs& d) {
    return splitmix64_dev(d.seed ^ ((unsigned long long)(*d.step) * 0x9E3779B97F4A7C15ULL) ^ ((unsigned long long)d.layer_id << 48));
}
__device__ __forceinline__ float drop_mult(unsigned long long key, unsigned int m, unsigned int n, float rate, float inv_keep) {
    const unsigned long long r = splitmix64_dev(key ^ ((unsigned long long)m * 65536ULL + n));
    const float u = (float)(unsigned int)(r >> 40) * (1.f / 16777216.f);
    return u >= rate ? inv_keep : 0.f;
}

// a hidden layer's output from its (dropped-out) post-activation value: the BN inference affine, gamma / sqrt(1 + 1e-3) and beta
// (tf.layers.batch_normalization with the initial moving statistics).  The FFMA forward epilogue, dropout_fwd_kernel and the
// layer summaries (summary.cu) all take it from here, so they agree bit for bit.
__device__ __forceinline__ float bn_out(float a, const float* __restrict__ gamma, const float* __restrict__ beta, int n, int bn) {
    return bn ? fmaf(a, gamma[n] * 0.99950037468777f, beta[n]) : a;
}

// hi = bf16(x) (round to nearest), lo = bf16(x - hi): x = hi + lo up to 2^-17 relative; the product a*b is rebuilt as
// a_lo*b_hi + a_hi*b_lo + a_hi*b_hi on the bf16 tensor pipe with fp32 accumulation (dropped term ~2^-18)
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// the same for two values at once, as packed bf16 pairs (x0 in the low half)
__device__ __forceinline__ void split_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    const __nv_bfloat162 hp = __floats2bfloat162_rn(x0, x1);
    hi = *reinterpret_cast<const uint32_t*>(&hp);
    const __nv_bfloat162 lp = __floats2bfloat162_rn(x0 - __uint_as_float(hi << 16), x1 - __uint_as_float(hi & 0xFFFF0000u));
    lo = *reinterpret_cast<const uint32_t*>(&lp);
}
// hi / lo copies of four consecutive values: one 8-byte store to each (hi and lo 8-byte aligned)
__device__ __forceinline__ void store_split4(__nv_bfloat16* hi, __nv_bfloat16* lo, float x0, float x1, float x2, float x3) {
    uint2 ph, pl;
    split_pair(x0, x1, ph.x, pl.x);
    split_pair(x2, x3, ph.y, pl.y);
    *reinterpret_cast<uint2*>(hi) = ph;
    *reinterpret_cast<uint2*>(lo) = pl;
}

}  // namespace wd
