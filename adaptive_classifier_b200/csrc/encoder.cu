// encoder.cu -- stage E: BERT / RoBERTa post-LN and ModernBERT pre-LN encoder forward -> unit-norm CLS rows.
//
// Replaces `self.model(**inputs).last_hidden_state[:, 0, :]` + F.normalize at
// /root/reference/src/adaptive_classifier/classifier.py:1271-1275 (HF BertModel.forward:
// embeddings modeling_bert.py:53-113, self-attention :143-207, output+LN :287-298, FFN :330-356;
// HF ModernBertModel.forward in models/modernbert/modeling_modernbert.py; NomicBertModel / JinaEmbeddingsV3Model, the
// post-LN block with RoPE and, for Nomic, a SwiGLU FFN; EuroBertModel, ModernBERT's pre-norm block with RMSNorm and SwiGLU).  One layer loop (forward_layers) runs both block kinds; they
// differ in the LayerNorm left pending on the residual path and in compile-time epilogue choices.
//
// Precision: every tensor-core operand is fp16 (RNE from fp32), accumulation fp32 (wgmma), residual stream, LayerNorm,
// softmax and GELU in fp32.  fp16 carries the same 10-bit mantissa as tf32, so the measured error is the tf32 one
// (oracle/precision_study.py: 1.7e-4 on squared-L2 distances, bf16 would be 1.4e-3 > the 1e-3 tolerance) at twice the
// tensor rate and half the operand bytes.
//
//   projections   wgmma GEMM of gemm_tc.cuh (.f16) with compile-time-specialised fused epilogues:
//                 bias | bias+GELU(erf or tanh) | bias+residual, fp16 or fp32 output, V written TRANSPOSED per (sequence, head);
//                 ALBERT / ELECTRA: LayerNorm at the embedding width E, then one E -> H projection (EpiEmbProj)
//   attention     one CTA per (sequence, head): Q, K and V^T tiles by TMA, QK^T and PV as wgmma with the score tile
//                 staged in shared memory, thread-per-query-row softmax in between (S <= 128; head_dim 64 or 32); longer
//                 sequences (up to 512, ModernBERT up to 8192) run 128-query blocks over streamed key blocks in one pass with
//                 an online softmax that visits only the key blocks inside a sliding layer's band (attention_stream_kernel);
//                 RoBERTa-arch encoders with a long position table (XLM-R, up to 8192) run full attention past 512 with the
//                 softmax on the wgmma fragments and P as the register A operand of the PV wgmma (attention_long_kernel)
//   LayerNorm     never materialised inside the layer stack: the residual epilogues keep the un-normalised sums y (fp32) and
//                 per-row (sum, sumsq) partials, the consuming projections run on gamma-scaled weights and apply the
//                 rank-1 correction r (acc - mu c1) + c0 in their epilogue ("deferred LayerNorm" below)
#include "gemm_tc.cuh"
#include <cuda_fp16.h>
#include <math_constants.h>
#include <algorithm>
#include <array>
#include <type_traits>
#include <vector>

namespace ac {

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// exact-erf GELU y*Phi(y) with erfc from Abramowitz-Stegun 7.1.26 (|error| < 1.5e-7 + 2 ulp of the two MUFU
// approximations).  With x = |y|/sqrt2, h = erfc(x)/2 = (poly(t)/2) * t * exp(-x^2), t = 1/(1 + p x):
//     y >= 0: y*(1 - h) = y - y*h        y < 0: y*h            =>   gelu(y) = max(y, 0) - |y*h|
// 2 MUFU + 12 FP32 ops per element and no branch/select.  The GELU epilogue touches 201 M elements per layer; the
// issue budget that hides it behind a K = 768 fp16 mainloop is ~24 instructions per element (libdevice erff alone ~30).
__device__ __forceinline__ float gelu_erf(float y) {
    const float ay = fabsf(y);
    const float t = rcp_approx(fmaf(0.3275911f * 0.70710678118654752440f, ay, 1.f));
    float p = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
    p = fmaf(p, t, 0.5f * 1.421413741f);
    p = fmaf(p, t, 0.5f * -0.284496736f);
    p = fmaf(p, t, 0.5f * 0.254829592f);
    const float e = ex2_approx((y * y) * (-0.5f * 1.4426950408889634f));   // exp(-y^2/2)
    const float h = (p * t) * e;                                             // erfc(|y|/sqrt2) / 2
    return fmaxf(y, 0.f) - fabsf(y * h);
}
// tanh-approximated GELU (HF "gelu_new" = "gelu_pytorch_tanh", ALBERT v2):  0.5 y (1 + tanh(u)) = y / (1 + exp(-2 u)),
// u = sqrt(2/pi) (y + 0.044715 y^3), with exp(-2 u) = 2^t, t = y (k1 + k3 y^2).  2 MUFU + 6 FP32 ops.  Relative error
// < 2^-15: k1 and k3 are formed in double and rounded once (1/2 ulp each, so the sum k1 + k3 y^2 carries at most 1/2 ulp of
// constant error); y^2, the fma and the product add 1/2 ulp each: |dt| <= 4 * 2^-24 |t|, an exp error <= 4 ln2 |t| 2^-24 <=
// 2.1e-5 for |t| <= 126, where 2^t stays finite (outputs that are normal fp16 need |t| <= ~30: <= 5e-6).  ex2.approx <= 2 ulp,
// rcp.approx <= 1 ulp, the add and the product 1/2 ulp each (< 5e-7 together).  Below t = -126 / above 126 the result is y / -0.
__device__ __forceinline__ float gelu_tanh(float y) {
    constexpr float k1 = static_cast<float>(-2.0 * 0.79788456080286535588 * 1.4426950408889634074);   // -2 sqrt(2/pi) log2(e)
    constexpr float k3 = static_cast<float>(-2.0 * 0.79788456080286535588 * 1.4426950408889634074 * 0.044715);
    const float t = y * fmaf(k3, y * y, k1);
    return y * rcp_approx(1.f + ex2_approx(t));
}
// SiLU (NomicBERT's SwiGLU, HF "silu" / "swish"):  y sigma(y) = y / (1 + exp(-y)) = y / (1 + 2^t), t = y k, k = -log2(e)
// rounded once from double.  2 MUFU + 3 FP32 ops.  Relative error: k and the product are 1/2 ulp each, |dt| <= 2 * 2^-24 |t|,
// an exp error <= 2 ln2 |t| 2^-24 (<= 1.0e-5 for |t| <= 126; the inputs with |y| <= 20 have |t| <= 29: <= 2.4e-6), damped by
// 2^t / (1 + 2^t) < 1 in the quotient; ex2.approx <= 2 ulp, the add 1/2 ulp, rcp.approx <= 1 ulp, the product 1/2 ulp
// (< 5e-7 together).  For y < -88.7 (t > 128) 2^t = +inf and the result is y * 0 = -0, never NaN; for t < -126 it is y.
__device__ __forceinline__ float silu(float y) {
    constexpr float k = static_cast<float>(-1.4426950408889634074);
    return y * rcp_approx(1.f + ex2_approx(y * k));
}

// ------------------------------------------------------------------------------------------------
// fused epilogues of the encoder linears (gemm_tc.cuh's epilogue concept), one type per projection role.  A thread holds
// one accumulator row; a warp's 32 rows leave through its staging tile as coalesced rows.  What they all share: the
// whole grid runs, no per-CTA state, both chunks of a tile unrolled (`buf` must be a compile-time constant).
struct EpiBase {
    static constexpr int kUnrollChunks = 4;
    __device__ __forceinline__ bool skip_kernel() const { return false; }
    template <class State> __device__ __forceinline__ void begin_cta(State &, int, int) const {}
    template <class State> __device__ __forceinline__ void end_cta(State &, int, int) const {}
};

// one 16-column half of this thread's 32 accumulators into row `lane` of the warp's staging tile; afterwards lane
// (r8 = lane / 4, c = lane % 4) reads the float4 of rows r8 + 8 i (i < 4) at byte 16 c
__device__ __forceinline__ void stage_f32_half(const float (&v)[32], int half, uint8_t *stage, int lane) {
    float4 *srow = reinterpret_cast<float4 *>(stage + lane * GEMM_EPI_STAGE_ROW_BYTES);
#pragma unroll
    for (int j = 0; j < 4; ++j)
        srow[j] = make_float4(v[16 * half + 4 * j], v[16 * half + 4 * j + 1], v[16 * half + 4 * j + 2], v[16 * half + 4 * j + 3]);
    __syncwarp();
}

__device__ __forceinline__ float gelu_if(bool on, float y) { return on ? gelu_erf(y) : y; }

// fp32 output: bias, then GELU (exact erf) or + fp32 residual; round_out rounds to tf32 (tests of the tf32 path)
template <bool GELU, bool RESID>
struct EpiF32 : EpiBase {
    const float *__restrict__ bias;       // [N]
    const float *__restrict__ residual;   // RESID: [M, ldy]
    float *Y;                             // [M, ldy]
    int M, N, ldy;
    int round_out = 0;
    // RESID requests each chunk's residual right before the chunk: one buffer of 32 registers instead of two keeps the
    // epilogue within the GEMM's 160 registers per thread
    static constexpr int kPrefetchDist = 0;
    struct State { float4 res[8]; };      // residual of one chunk: [column half][row pass], the staged layout
    __device__ __forceinline__ void prefetch(State &st, const GemmTileInfo &, int row, int col0, int lane, int) const {
        if (!RESID) return;
        const int row_base = row - lane;
        const int r8 = lane >> 2, c = lane & 3;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int col = col0 + 16 * half + 4 * c;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int grow = row_base + r8 + 8 * i;
                st.res[half * 4 + i] =
                    (grow < M && col + 4 <= N)
                        ? __ldg(reinterpret_cast<const float4 *>(residual + static_cast<int64_t>(grow) * ldy + col))
                        : make_float4(0, 0, 0, 0);
            }
        }
    }
    __device__ __forceinline__ void tile(State &st, const GemmTileInfo &, int row, int col0, const float (&v)[32], uint8_t *stage,
                                         int lane, int, const float *) const {
        const int row_base = row - lane;                                     // first row of this warp's quarter
        if (row_base >= M || col0 >= N) return;                              // warp-uniform
        const int r8 = lane >> 2, c = lane & 3;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int col = col0 + 16 * half + 4 * c;
            stage_f32_half(v, half, stage, lane);
            const float4 b4 = (col + 4 <= N) ? __ldg(reinterpret_cast<const float4 *>(bias + col)) : make_float4(0, 0, 0, 0);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int rr = r8 + 8 * i;
                const int grow = row_base + rr;
                if (grow < M && col + 4 <= N) {
                    const float4 a = *reinterpret_cast<const float4 *>(stage + rr * GEMM_EPI_STAGE_ROW_BYTES + 16 * c);
                    float4 o;
                    o.x = gelu_if(GELU, a.x + b4.x); o.y = gelu_if(GELU, a.y + b4.y);
                    o.z = gelu_if(GELU, a.z + b4.z); o.w = gelu_if(GELU, a.w + b4.w);
                    if (RESID) {
                        const float4 rs = st.res[half * 4 + i];                 // requested before the chunk
                        o.x += rs.x; o.y += rs.y; o.z += rs.z; o.w += rs.w;
                    }
                    if (round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
                    *reinterpret_cast<float4 *>(Y + static_cast<int64_t>(grow) * ldy + col) = o;
                }
            }
            __syncwarp();
        }
    }
};

// fp16 output, the next GEMM's A operand: pre-activation acc + bias, or with DEFER the deferred-LayerNorm form below, then
//   Act::Gelu   exact-erf GELU
//   Act::GeluTanh  tanh-approximated GELU (post-LN encoders with hidden_act "gelu_new" / "gelu_pytorch_tanh")
//   Act::GeGLU  (ModernBERT's mlp.Wi) pack_defer_kernel interleaved the weight rows in 32-row groups, so a warp's slice
//               holds [input cols 32 g .. + 31 | gate cols 32 g .. + 31]; the gate chunk re-reads the input chunk from the
//               accumulator tile and writes fp16(GELU_erf(input) * gate) to columns 32 g.. of Y (N = 2 I, ldy = I)
//   Act::SwiGLU (NomicBERT's gate_proj | up_proj) GeGLU's layout and path with silu: fp16(silu(gate_proj) * up_proj)
//   Act::Rope   (q and k of ModernBERT's Wqkv) rotated in fp32 before the fp16 rounding: the pair (d, d + 32) of a head is
//               the two chunks of a warp's slice, the partner re-read from the accumulator tile; position = row % S
// DEFER: the A operand was the UN-normalised residual sum y (fp16) and the weights were packed as fp16(gamma * W):
//   LayerNorm(y) W^T + b = r (acc - mu c1) + c0  with the row statistics (mu, r) of y, c1 = rowsum(W'), and `bias`
//   holding c0 = W beta + b  (producer side: EpiResidDefer)
enum class Act { None, Gelu, GeGLU, Rope, GeluTanh, SwiGLU };
// the activation an EpiF16 applies to every pre-activation (GeGLU and RoPE combine a chunk with its partner instead)
template <Act ACT>
__device__ __forceinline__ float act_elem(float y) {
    if constexpr (ACT == Act::Gelu) return gelu_erf(y);
    else if constexpr (ACT == Act::GeluTanh) return gelu_tanh(y);
    else return y;
}
template <Act ACT, bool DEFER>
struct EpiF16 : EpiBase {
    const float *__restrict__ bias;       // [N]   (DEFER: c0)
    const float *__restrict__ c1;         // DEFER: [N] row sums of the packed weight
    const float2 *__restrict__ row_stats; // DEFER: [M] (mu, 1/sqrt(var + eps)) of the A rows
    __half *Y;                            // [M, ldy]
    int M, N, ldy;
    int S;                                // Act::Rope, EpiQKV: tokens per sequence
    const float *__restrict__ rope;       // Act::Rope: [S, 64] cos | sin per position
    static constexpr int kPrefetchDist = 1;   // DEFER: the row statistics are requested before the accumulators arrive
    struct State { float mu, r; };            // DEFER: statistics of this thread's accumulator row
    __device__ __forceinline__ float pre(const State &st, float acc, float b, float c1v) const {
        return DEFER ? fmaf(st.r, fmaf(-st.mu, c1v, acc), b) : acc + b;
    }
    __device__ __forceinline__ void prefetch(State &st, const GemmTileInfo &ti, int row, int col0, int, int) const {
        if (DEFER && ((col0 - ti.n0) & (GEMM_EPI_COLS - 1)) == 0) {    // first chunk of this warp's column slice
            const float2 ms = (row < M) ? __ldg(row_stats + row) : make_float2(0.f, 0.f);
            st.mu = ms.x, st.r = ms.y;
        }
    }
    __device__ __forceinline__ void tile(State &st, const GemmTileInfo &, int row, int col0, const float (&v)[32], uint8_t *stage,
                                         int lane, int, const float *acc) const {
        const int row_base = row - lane;                                     // first row of this warp's quarter
        if (row_base >= M || col0 >= N) return;                              // warp-uniform
        constexpr bool GLU = ACT == Act::GeGLU || ACT == Act::SwiGLU, ROT = ACT == Act::Rope;
        if (GLU && (col0 & 32) == 0) return;                                 // input chunk: consumed by its gate chunk
        const int ocol0 = GLU ? (col0 - 32) / 2 : col0, oN = GLU ? N / 2 : N;
        const int pofs = (col0 & 32) ? -32 : 32;                             // partner chunk (RoPE half / GeGLU input)
        const float *rrow = ROT ? rope + static_cast<int64_t>(row < M ? row % S : 0) * 64 : nullptr;
        // stage 32 rows x 32 halves (64 B payload per 80-byte row), then lane (r4 = lane/4 .. 8 rows per pass, c8 = lane%4)
        uint4 *srow = reinterpret_cast<uint4 *>(stage + lane * GEMM_EPI_STAGE_ROW_BYTES);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float4 ba = __ldg(reinterpret_cast<const float4 *>(bias + col0 + 8 * j));
            const float4 bb = __ldg(reinterpret_cast<const float4 *>(bias + col0 + 8 * j + 4));
            const float4 ca = DEFER ? __ldg(reinterpret_cast<const float4 *>(c1 + col0 + 8 * j)) : make_float4(0, 0, 0, 0);
            const float4 cb = DEFER ? __ldg(reinterpret_cast<const float4 *>(c1 + col0 + 8 * j + 4)) : make_float4(0, 0, 0, 0);
            float y[8];
            y[0] = act_elem<ACT>(pre(st, v[8 * j], ba.x, ca.x)); y[1] = act_elem<ACT>(pre(st, v[8 * j + 1], ba.y, ca.y));
            y[2] = act_elem<ACT>(pre(st, v[8 * j + 2], ba.z, ca.z)); y[3] = act_elem<ACT>(pre(st, v[8 * j + 3], ba.w, ca.w));
            y[4] = act_elem<ACT>(pre(st, v[8 * j + 4], bb.x, cb.x)); y[5] = act_elem<ACT>(pre(st, v[8 * j + 5], bb.y, cb.y));
            y[6] = act_elem<ACT>(pre(st, v[8 * j + 6], bb.z, cb.z)); y[7] = act_elem<ACT>(pre(st, v[8 * j + 7], bb.w, cb.w));
            if (GLU || ROT) {
                const int pc = col0 + pofs + 8 * j;
                const float4 a0 = *reinterpret_cast<const float4 *>(acc + pofs + 8 * j);
                const float4 a1 = *reinterpret_cast<const float4 *>(acc + pofs + 8 * j + 4);
                const float4 pba = __ldg(reinterpret_cast<const float4 *>(bias + pc));
                const float4 pbb = __ldg(reinterpret_cast<const float4 *>(bias + pc + 4));
                const float4 pca = DEFER ? __ldg(reinterpret_cast<const float4 *>(c1 + pc)) : make_float4(0, 0, 0, 0);
                const float4 pcb = DEFER ? __ldg(reinterpret_cast<const float4 *>(c1 + pc + 4)) : make_float4(0, 0, 0, 0);
                float p[8];
                p[0] = pre(st, a0.x, pba.x, pca.x); p[1] = pre(st, a0.y, pba.y, pca.y);
                p[2] = pre(st, a0.z, pba.z, pca.z); p[3] = pre(st, a0.w, pba.w, pca.w);
                p[4] = pre(st, a1.x, pbb.x, pcb.x); p[5] = pre(st, a1.y, pbb.y, pcb.y);
                p[6] = pre(st, a1.z, pbb.z, pcb.z); p[7] = pre(st, a1.w, pbb.w, pcb.w);
                if (GLU) {
#pragma unroll
                    for (int k = 0; k < 8; ++k)                                         // y = gate, p = input
                        y[k] = (ACT == Act::SwiGLU ? silu(p[k]) : gelu_erf(p[k])) * y[k];
                } else {
                    // HF apply_rotary_pos_emb: x cos + rotate_half(x) sin, rotate_half = (-x[32:], x[:32])
                    const float4 c0v = __ldg(reinterpret_cast<const float4 *>(rrow + 8 * j));
                    const float4 c1v = __ldg(reinterpret_cast<const float4 *>(rrow + 8 * j + 4));
                    const float4 s0v = __ldg(reinterpret_cast<const float4 *>(rrow + 32 + 8 * j));
                    const float4 s1v = __ldg(reinterpret_cast<const float4 *>(rrow + 32 + 8 * j + 4));
                    const float cs[8] = {c0v.x, c0v.y, c0v.z, c0v.w, c1v.x, c1v.y, c1v.z, c1v.w};
                    const float sn[8] = {s0v.x, s0v.y, s0v.z, s0v.w, s1v.x, s1v.y, s1v.z, s1v.w};
                    const float sg = (col0 & 32) ? 1.f : -1.f;
#pragma unroll
                    for (int k = 0; k < 8; ++k) y[k] = __fadd_rn(__fmul_rn(y[k], cs[k]), __fmul_rn(sg * p[k], sn[k]));
                }
            }
            uint4 pk;
            __half2 h0 = __floats2half2_rn(y[0], y[1]), h1 = __floats2half2_rn(y[2], y[3]);
            __half2 h2 = __floats2half2_rn(y[4], y[5]), h3 = __floats2half2_rn(y[6], y[7]);
            pk.x = *reinterpret_cast<uint32_t *>(&h0); pk.y = *reinterpret_cast<uint32_t *>(&h1);
            pk.z = *reinterpret_cast<uint32_t *>(&h2); pk.w = *reinterpret_cast<uint32_t *>(&h3);
            srow[j] = pk;
        }
        __syncwarp();
        const int r8 = lane >> 2, c = lane & 3;                               // 8 rows x 4 x 16 B per pass
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int rr = r8 + 8 * i;
            const int grow = row_base + rr;
            const int col = ocol0 + 8 * c;
            if (grow < M && col + 8 <= oN) {
                const uint4 pk = *reinterpret_cast<const uint4 *>(stage + rr * GEMM_EPI_STAGE_ROW_BYTES + 16 * c);
                *reinterpret_cast<uint4 *>(Y + static_cast<int64_t>(grow) * ldy + col) = pk;
            }
        }
        __syncwarp();
    }
};

// fused QKV, a deferred-LayerNorm consumer: q and k (columns < vt_col0) are EpiF16 rows (ModernBERT: RoPE); V is written
// transposed to vT[(b*H + feature) * S_pad + key] so that attention can TMA-load V^T as a K-major B operand.
template <bool ROPE>
struct EpiQKV : EpiBase {
    EpiF16<ROPE ? Act::Rope : Act::None, true> qk;   // N = 3 H accumulator columns, Y = [M, 2 H] q | k
    __half *vT;
    int vt_col0, S_pad, H;
    static constexpr int kPrefetchDist = 1;
    using State = typename decltype(qk)::State;
    __device__ __forceinline__ void prefetch(State &st, const GemmTileInfo &ti, int row, int col0, int lane, int buf) const {
        qk.prefetch(st, ti, row, col0, lane, buf);
    }
    __device__ __forceinline__ void tile(State &st, const GemmTileInfo &ti, int row, int col0, const float (&v)[32],
                                         uint8_t *stage, int lane, int buf, const float *acc) const {
        if (row - lane >= qk.M || col0 >= qk.N) return;                     // warp-uniform
        if (col0 < vt_col0) return qk.tile(st, ti, row, col0, v, stage, lane, buf, acc);
        // thread = token row: lanes hold 32 consecutive keys of (mostly) one sequence -> 64-byte coalesced stores
        if (row < qk.M) {
            const int b = row / qk.S, key = row - b * qk.S;
            __half *dst = vT + (static_cast<int64_t>(b) * H + (col0 - vt_col0)) * S_pad + key;
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                const float4 b4 = __ldg(reinterpret_cast<const float4 *>(qk.bias + col0 + j));
                const float4 c4 = __ldg(reinterpret_cast<const float4 *>(qk.c1 + col0 + j));
                dst[static_cast<int64_t>(j) * S_pad] = __float2half_rn(qk.pre(st, v[j], b4.x, c4.x));
                dst[static_cast<int64_t>(j + 1) * S_pad] = __float2half_rn(qk.pre(st, v[j + 1], b4.y, c4.y));
                dst[static_cast<int64_t>(j + 2) * S_pad] = __float2half_rn(qk.pre(st, v[j + 2], b4.z, c4.z));
                dst[static_cast<int64_t>(j + 3) * S_pad] = __float2half_rn(qk.pre(st, v[j + 3], b4.w, c4.w));
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------
// deferred LayerNorm: residual epilogue that never materialises LayerNorm
//   y_new = acc + bias + LN_prev(y_old)          LN_prev(y) = (y - mu) r gamma + beta recomputed from the fp32 y_old, its
//                                                row statistics and the pending LayerNorm's parameters
//   writes y_new (fp32, IN PLACE over y_old: every element is read and written by the same thread), fp16(y_new) (the
//   next GEMM's A operand, consumed through EpiF16<.., DEFER = true>) and per-row partial (sum, sum of squares) of
//   this warp's GEMM_EPI_COLS columns into parts[column part][row]; ln_stats_kernel turns the parts into (mu, r).
//   HBM traffic per half layer at B*S = 65536, H = 768: read y 201 MB, write y 201 MB + fp16 101 MB = 503 MB instead of
//   905 MB (GEMM epilogue 402 MB + LayerNorm kernel 503 MB); precision: oracle/deferred_ln_study.py (CPU emulation) and tests/test_gpu_parity.py (non-trivial gamma / beta).
// ------------------------------------------------------------------------------------------------
struct EpiResidDefer : EpiBase {
    const float *__restrict__ bias;        // [N]
    float *y;                              // [M, ld] fp32 residual sums: read (old) and written (new) in place
    __half *yh;                            // [M, ld] fp16 copy of the new sums
    const float2 *__restrict__ stats_prev; // [M] (mu, r) of the old sums
    const float *__restrict__ gamma;       // [N] pending LayerNorm of the old sums
    const float *__restrict__ beta;        // [N]
    float2 *parts;                         // [N / GEMM_EPI_COLS][part_stride] partial (sum, sumsq) of the new sums
    int64_t part_stride;
    int M, N, ld;
    // The residual epilogues are HBM-bound (fp32 sums read + written, fp16 copy written per element).  The old sums of the
    // next 32-column chunk are requested one chunk ahead; a larger distance needs one more 32-register buffer per thread.
    static constexpr int kPrefetchDist = 1;
    struct State {
        float4 res[kPrefetchDist + 1][8];  // old sums of 32-column chunks (transposed-phase layout), one buffer more than the distance
        float sum[4], sq[4];               // running partials of the new sums over this warp's GEMM_EPI_COLS columns
    };
    __device__ __forceinline__ void prefetch(State &st, const GemmTileInfo &ti, int row, int col0, int lane, int buf) const {
        const int row_base = row - lane;
        const int r8 = lane >> 2, c = lane & 3;
        if (((col0 - ti.n0) & (GEMM_EPI_COLS - 1)) == 0) {              // first chunk of this warp's column half
#pragma unroll
            for (int i = 0; i < 4; ++i) st.sum[i] = st.sq[i] = 0.f;
        }
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int col = col0 + 16 * half + 4 * c;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int grow = row_base + r8 + 8 * i;
                // plain (coherent) load: y is written by this very kernel, although never the element being read here
                st.res[buf][half * 4 + i] = (grow < M && col + 4 <= N)
                                                ? *reinterpret_cast<const float4 *>(y + static_cast<int64_t>(grow) * ld + col)
                                                : make_float4(0, 0, 0, 0);
            }
        }
    }
    __device__ __forceinline__ void tile(State &st, const GemmTileInfo &ti, int row, int col0, const float (&v)[32], uint8_t *stage,
                                         int lane, int buf, const float *) const {
        const int row_base = row - lane;
        if (row_base >= M || col0 >= N) return;                              // warp-uniform
        const int r8 = lane >> 2, c = lane & 3;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int col = col0 + 16 * half + 4 * c;
            stage_f32_half(v, half, stage, lane);
            const bool col_ok = col + 4 <= N;
            const float4 b4 = col_ok ? __ldg(reinterpret_cast<const float4 *>(bias + col)) : make_float4(0, 0, 0, 0);
            const float4 g4 = col_ok ? __ldg(reinterpret_cast<const float4 *>(gamma + col)) : make_float4(0, 0, 0, 0);
            const float4 e4 = col_ok ? __ldg(reinterpret_cast<const float4 *>(beta + col)) : make_float4(0, 0, 0, 0);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int rr = r8 + 8 * i;
                const int grow = row_base + rr;
                if (grow < M && col_ok) {
                    const float4 a = *reinterpret_cast<const float4 *>(stage + rr * GEMM_EPI_STAGE_ROW_BYTES + 16 * c);
                    const float4 rs = st.res[buf][half * 4 + i];             // old sums, requested one chunk ago
                    const float2 ms = __ldg(stats_prev + grow);             // (mu, r): re-read, not held across chunks
                    const float mu = ms.x, r = ms.y;
                    float4 o;
                    o.x = (a.x + b4.x) + fmaf((rs.x - mu) * r, g4.x, e4.x);
                    o.y = (a.y + b4.y) + fmaf((rs.y - mu) * r, g4.y, e4.y);
                    o.z = (a.z + b4.z) + fmaf((rs.z - mu) * r, g4.z, e4.z);
                    o.w = (a.w + b4.w) + fmaf((rs.w - mu) * r, g4.w, e4.w);
                    *reinterpret_cast<float4 *>(y + static_cast<int64_t>(grow) * ld + col) = o;
                    const __half2 h0 = __floats2half2_rn(o.x, o.y), h1 = __floats2half2_rn(o.z, o.w);
                    uint2 pk;
                    pk.x = *reinterpret_cast<const uint32_t *>(&h0);
                    pk.y = *reinterpret_cast<const uint32_t *>(&h1);
                    *reinterpret_cast<uint2 *>(yh + static_cast<int64_t>(grow) * ld + col) = pk;
                    st.sum[i] += (o.x + o.y) + (o.z + o.w);
                    st.sq[i] += (o.x * o.x + o.y * o.y) + (o.z * o.z + o.w * o.w);
                }
            }
            __syncwarp();
        }
        if (((col0 - ti.n0) & (GEMM_EPI_COLS - 1)) == GEMM_EPI_COLS - 32) {   // last chunk of this warp's column half
            const int part = col0 / GEMM_EPI_COLS;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float s = st.sum[i], q = st.sq[i];
                s += __shfl_xor_sync(0xffffffffu, s, 1);
                q += __shfl_xor_sync(0xffffffffu, q, 1);
                s += __shfl_xor_sync(0xffffffffu, s, 2);
                q += __shfl_xor_sync(0xffffffffu, q, 2);
                const int grow = row_base + r8 + 8 * i;
                if (c == 0 && grow < M) parts[static_cast<int64_t>(part) * part_stride + grow] = make_float2(s, q);
            }
        }
    }
};

// embedding projection E -> H (ALBERT encoder.embedding_hidden_mapping_in, ELECTRA embeddings_project): the A operand is
// the LayerNorm-ed embedding rows at width E (fp16), the output the residual stream layer 0 starts from, y = acc + bias in
// fp32 plus its fp16 copy yh (layer 0's QKV operand).  Nothing is pending on y: layer 0 runs with the identity LayerNorm,
// as it does on the embeddings of an encoder without projection.
struct EpiEmbProj : EpiBase {
    const float *__restrict__ bias;   // [N]
    float *y;                         // [M, ld]
    __half *yh;                       // [M, ld]
    int M, N, ld;
    static constexpr int kPrefetchDist = 0;
    struct State {};
    __device__ __forceinline__ void prefetch(State &, const GemmTileInfo &, int, int, int, int) const {}
    __device__ __forceinline__ void tile(State &, const GemmTileInfo &, int row, int col0, const float (&v)[32], uint8_t *stage,
                                         int lane, int, const float *) const {
        const int row_base = row - lane;
        if (row_base >= M || col0 >= N) return;                              // warp-uniform
        const int r8 = lane >> 2, c = lane & 3;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int col = col0 + 16 * half + 4 * c;
            stage_f32_half(v, half, stage, lane);
            const bool col_ok = col + 4 <= N;
            const float4 b4 = col_ok ? __ldg(reinterpret_cast<const float4 *>(bias + col)) : make_float4(0, 0, 0, 0);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int grow = row_base + r8 + 8 * i;
                if (grow < M && col_ok) {
                    const float4 a = *reinterpret_cast<const float4 *>(stage + (r8 + 8 * i) * GEMM_EPI_STAGE_ROW_BYTES + 16 * c);
                    const float4 o = make_float4(a.x + b4.x, a.y + b4.y, a.z + b4.z, a.w + b4.w);
                    *reinterpret_cast<float4 *>(y + static_cast<int64_t>(grow) * ld + col) = o;
                    const __half2 h0 = __floats2half2_rn(o.x, o.y), h1 = __floats2half2_rn(o.z, o.w);
                    uint2 pk;
                    pk.x = *reinterpret_cast<const uint32_t *>(&h0);
                    pk.y = *reinterpret_cast<const uint32_t *>(&h1);
                    *reinterpret_cast<uint2 *>(yh + static_cast<int64_t>(grow) * ld + col) = pk;
                }
            }
            __syncwarp();
        }
    }
};

// The norm a block applies to its residual sums: LayerNorm (BERT family, ModernBERT) or RMSNorm (EuroBERT: weight * y /
// sqrt(mean(y^2) + eps), no mean subtraction, no bias).  A deferred RMSNorm is the deferred LayerNorm with row statistics
// (0, 1/sqrt(mean(y^2) + eps)) and beta 0, so every deferred-norm epilogue serves both.
enum class Norm { Layer, Rms };

// (sum, sumsq) partials of every GEMM_EPI_COLS-column part -> (mu, 1/sqrt(var + eps)) per row (RMS: (0, 1/sqrt(sumsq/H + eps)));
// parts are added in a fixed order.
// Kept as a kernel of its own: folding these loads + rsqrt into the consuming epilogues puts them at the head of every tile's
// epilogue, which is the critical path of the HBM-bound residual GEMMs.
template <Norm NORM>
__global__ void ln_stats_kernel(const float2 *__restrict__ parts, int nparts, int64_t part_stride, int rows, int H, float eps,
                                float2 *__restrict__ stats) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= rows) return;
    float s = 0.f, q = 0.f;
    for (int p = 0; p < nparts; ++p) {
        const float2 v = parts[static_cast<int64_t>(p) * part_stride + row];
        s += v.x;
        q += v.y;
    }
    if constexpr (NORM == Norm::Rms) {
        stats[row] = make_float2(0.f, 1.f / sqrtf(q / static_cast<float>(H) + eps));
        return;
    }
    const float mu = s / static_cast<float>(H);
    const float var = fmaxf(q / static_cast<float>(H) - mu * mu, 0.f);
    stats[row] = make_float2(mu, 1.f / sqrtf(var + eps));
}

__global__ void fill_stats_identity_kernel(float2 *__restrict__ stats, int64_t n) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) stats[i] = make_float2(0.f, 1.f);
}
__global__ void fill_value_kernel(float *__restrict__ p, int n, float v) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// weight packing of a deferred-LayerNorm consumer (one warp per output row n):
//   Wp[n,k] = fp16(gamma[k] W[n,k]),  c1[n] = sum_k Wp[n,k] (fp32),  c0[n] = sum_k beta[k] W[n,k] + bias[n]
// gamma / beta NULL = identity LayerNorm (layer 0 consumes the already normalised embeddings), bias NULL = 0.
// glu != 0 (GeGLU weight [2I, H], N = 2I): packed row n takes source row (n / 64) 32 + n % 32 of the input half for
// n % 64 < 32, the same row of the gate half otherwise -- the row order EpiF16<Act::GeGLU / Act::SwiGLU, ..> expects
__global__ void pack_defer_kernel(const float *__restrict__ W, const float *__restrict__ bias, const float *__restrict__ gamma,
                                  const float *__restrict__ beta, int N, int K, __half *__restrict__ Wp, float *__restrict__ c1,
                                  float *__restrict__ c0, int glu = 0) {
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= N) return;
    const int src = glu ? (n >> 6) * 32 + (n & 31) + ((n & 32) ? N / 2 : 0) : n;
    float s1 = 0.f, s0 = 0.f;
    for (int k = lane; k < K; k += 32) {
        const float w = W[static_cast<int64_t>(src) * K + k];
        const __half h = __float2half_rn(gamma ? gamma[k] * w : w);
        Wp[static_cast<int64_t>(n) * K + k] = h;
        s1 += __half2float(h);
        s0 = fmaf(beta ? beta[k] : 0.f, w, s0);
    }
    s1 = warp_sum(s1);
    s0 = warp_sum(s0);
    if (lane == 0) {
        c1[n] = s1;
        c0[n] = s0 + (bias ? bias[src] : 0.f);
    }
}

// ------------------------------------------------------------------------------------------------
// elementwise / normalisation kernels (one warp per row, float4 lanes; H % 128 == 0, H <= 1024)
// ------------------------------------------------------------------------------------------------
constexpr int LN_MAXV = 8;

// RMS: weight * (x / sqrt(mean(x^2) + eps)) (EuroBertRMSNorm, fp32); b is not read
template <Norm NORM = Norm::Layer>
__device__ __forceinline__ void ln_row(float4 (&x)[LN_MAXV], int nv, int H, const float *__restrict__ w,
                                       const float *__restrict__ b, float eps, int lane, float *out_full,
                                       __half *out_half) {
    if constexpr (NORM == Norm::Rms) {
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < LN_MAXV; ++i)
            if (i < nv) q += (x[i].x * x[i].x + x[i].y * x[i].y) + (x[i].z * x[i].z + x[i].w * x[i].w);
        const float r = 1.f / sqrtf(warp_sum(q) / static_cast<float>(H) + eps);
#pragma unroll
        for (int i = 0; i < LN_MAXV; ++i)
            if (i < nv) {
                const int col = (lane + 32 * i) * 4;
                const float4 w4 = __ldg(reinterpret_cast<const float4 *>(w + col));
                const float4 o = make_float4(x[i].x * r * w4.x, x[i].y * r * w4.y, x[i].z * r * w4.z, x[i].w * r * w4.w);
                if (out_full) *reinterpret_cast<float4 *>(out_full + col) = o;
                if (out_half) {
                    __half2 h0 = __floats2half2_rn(o.x, o.y), h1 = __floats2half2_rn(o.z, o.w);
                    uint2 pk;
                    pk.x = *reinterpret_cast<uint32_t *>(&h0);
                    pk.y = *reinterpret_cast<uint32_t *>(&h1);
                    *reinterpret_cast<uint2 *>(out_half + col) = pk;
                }
            }
        return;
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (i < nv) s += (x[i].x + x[i].y) + (x[i].z + x[i].w);
    const float mean = warp_sum(s) / static_cast<float>(H);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (i < nv) {
            const float a = x[i].x - mean, c = x[i].y - mean, d = x[i].z - mean, e = x[i].w - mean;
            q += (a * a + c * c) + (d * d + e * e);
        }
    const float var = warp_sum(q) / static_cast<float>(H);
    const float rstd = 1.f / sqrtf(var + eps);
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (i < nv) {
            const int col = (lane + 32 * i) * 4;
            const float4 w4 = __ldg(reinterpret_cast<const float4 *>(w + col));
            const float4 b4 = __ldg(reinterpret_cast<const float4 *>(b + col));
            float4 o;
            o.x = (x[i].x - mean) * rstd * w4.x + b4.x;
            o.y = (x[i].y - mean) * rstd * w4.y + b4.y;
            o.z = (x[i].z - mean) * rstd * w4.z + b4.z;
            o.w = (x[i].w - mean) * rstd * w4.w + b4.w;
            if (out_full) *reinterpret_cast<float4 *>(out_full + col) = o;
            if (out_half) {
                __half2 h0 = __floats2half2_rn(o.x, o.y), h1 = __floats2half2_rn(o.z, o.w);
                uint2 pk;
                pk.x = *reinterpret_cast<uint32_t *>(&h0);
                pk.y = *reinterpret_cast<uint32_t *>(&h1);
                *reinterpret_cast<uint2 *>(out_half + col) = pk;
            }
        }
}

template <Norm NORM>
__global__ void layernorm_kernel(const float *__restrict__ in, const float *__restrict__ w, const float *__restrict__ b,
                                 float eps, int rows, int H, float *__restrict__ out_full, __half *__restrict__ out_half) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int nv = H / 128;
    float4 x[LN_MAXV];
    const float *src = in + static_cast<int64_t>(row) * H;
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (i < nv) x[i] = *reinterpret_cast<const float4 *>(src + (lane + 32 * i) * 4);
    ln_row<NORM>(x, nv, H, w, b, eps, lane, out_full ? out_full + static_cast<int64_t>(row) * H : nullptr,
                 out_half ? out_half + static_cast<int64_t>(row) * H : nullptr);
}

// modeling_bert.py:53-113 / modeling_roberta.py:146-159: (word + type) + position -> LayerNorm
// modeling_mpnet.py MPNetEmbeddings: RoBERTa's positions (padding_idx 1); the type table is one zero row
// modeling_modernbert.py ModernBertEmbeddings: pos = type = NULL, LayerNorm(word) (b = zeros: norm_bias=False)
// modeling_albert.py AlbertEmbeddings, modeling_electra.py ElectraEmbeddings: BERT's rule at width H = embedding_size;
// F32_OUT = false writes the fp16 rows only (the A operand of the embedding projection, EpiEmbProj)
// RAW_RMS (modeling_eurobert.py EuroBertModel: embed_tokens(ids), no norm, no position table; pos = NULL): the raw word row
// is the residual stream (out_full, out_half) and rms_stats[row] = (0, 1/sqrt(mean(x^2) + eps)) are the statistics of
// layer 0's deferred input_layernorm; w, b are not read
template <bool F32_OUT, bool RAW_RMS = false>
__global__ void embed_ln_kernel(const int32_t *__restrict__ ids, const int32_t *__restrict__ type_ids,
                                const float *__restrict__ word, const float *__restrict__ pos,
                                const float *__restrict__ type, const float *__restrict__ w,
                                const float *__restrict__ b, float eps, int B, int S, int H, int arch, int pad_idx,
                                int vocab, int max_pos, int type_vocab, float *__restrict__ out_full,
                                __half *__restrict__ out_half, float2 *__restrict__ rms_stats = nullptr) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= B * S) return;
    const int bq = row / S, s = row % S;
    int id = ids[row];
    id = min(max(id, 0), vocab - 1);
    int tt = type_ids ? type_ids[row] : 0;
    tt = min(max(tt, 0), type_vocab - 1);
    int p = s;
    if (arch == AC_ARCH_ROBERTA || arch == AC_ARCH_MPNET) {
        // position = cumsum(ids != pad)[s] * (id != pad) + pad_idx
        int cnt = 0;
        for (int j = lane; j <= s; j += 32) cnt += (ids[bq * S + j] != pad_idx) ? 1 : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        p = (id != pad_idx) ? cnt + pad_idx : pad_idx;
    }
    p = min(p, max_pos - 1);
    const int nv = H / 128;
    float4 x[LN_MAXV];
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (i < nv) {
            const int col = (lane + 32 * i) * 4;
            const float4 a = __ldg(reinterpret_cast<const float4 *>(word + static_cast<int64_t>(id) * H + col));
            if (!pos) {
                x[i] = a;
                continue;
            }
            const float4 t = __ldg(reinterpret_cast<const float4 *>(type + static_cast<int64_t>(tt) * H + col));
            const float4 q = __ldg(reinterpret_cast<const float4 *>(pos + static_cast<int64_t>(p) * H + col));
            x[i].x = (a.x + t.x) + q.x;
            x[i].y = (a.y + t.y) + q.y;
            x[i].z = (a.z + t.z) + q.z;
            x[i].w = (a.w + t.w) + q.w;
        }
    if constexpr (RAW_RMS) {
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < LN_MAXV; ++i)
            if (i < nv) {
                const int col = (lane + 32 * i) * 4;
                *reinterpret_cast<float4 *>(out_full + static_cast<int64_t>(row) * H + col) = x[i];
                const __half2 h0 = __floats2half2_rn(x[i].x, x[i].y), h1 = __floats2half2_rn(x[i].z, x[i].w);
                uint2 pk;
                pk.x = *reinterpret_cast<const uint32_t *>(&h0);
                pk.y = *reinterpret_cast<const uint32_t *>(&h1);
                *reinterpret_cast<uint2 *>(out_half + static_cast<int64_t>(row) * H + col) = pk;
                q += (x[i].x * x[i].x + x[i].y * x[i].y) + (x[i].z * x[i].z + x[i].w * x[i].w);
            }
        q = warp_sum(q);
        if (lane == 0) rms_stats[row] = make_float2(0.f, 1.f / sqrtf(q / static_cast<float>(H) + eps));
        return;
    }
    ln_row(x, nv, H, w, b, eps, lane, F32_OUT ? out_full + static_cast<int64_t>(row) * H : nullptr,
           out_half + static_cast<int64_t>(row) * H);
}

// classifier.py:1272,1275: CLS row -> x / max(||x||_2, 1e-12)
__global__ void cls_normalize_kernel(const float *__restrict__ x, int B, int S, int H, float *__restrict__ out) {
    const int bq = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (bq >= B) return;
    const float *src = x + static_cast<int64_t>(bq) * S * H;
    float s = 0.f;
    for (int i = lane; i < H; i += 32) s = fmaf(src[i], src[i], s);
    const float nrm = fmaxf(sqrtf(warp_sum(s)), 1e-12f);
    for (int i = lane; i < H; i += 32) out[static_cast<int64_t>(bq) * H + i] = src[i] / nrm;
}

// last layer: only the CLS row of every sequence is needed downstream of attention (classifier.py:1272), so the
// output projection, both LayerNorms and the FFN of the last layer run on B rows instead of B*S
__global__ void gather_cls_kernel(const __half *__restrict__ ctx, const float *__restrict__ x, int B, int S, int H,
                                  __half *__restrict__ ctx_cls, float *__restrict__ x_cls) {
    const int bq = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (bq >= B) return;
    const int64_t src = static_cast<int64_t>(bq) * S * H, dst = static_cast<int64_t>(bq) * H;
    for (int i = lane; i < H / 8; i += 32)
        reinterpret_cast<uint4 *>(ctx_cls + dst)[i] = reinterpret_cast<const uint4 *>(ctx + src)[i];
    for (int i = lane; i < H / 4; i += 32)
        reinterpret_cast<float4 *>(x_cls + dst)[i] = reinterpret_cast<const float4 *>(x + src)[i];
}

__global__ void round_copy_kernel(const float *__restrict__ in, float *__restrict__ out, int64_t n, int do_round) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = do_round ? round_tf32(in[i]) : in[i];
}
__global__ void to_half_kernel(const float *__restrict__ in, __half *__restrict__ out, int64_t n) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = __float2half_rn(in[i]);
}

// ------------------------------------------------------------------------------------------------
// attention: one CTA (128 threads = one warpgroup) per (sequence b, head h); S <= 128, head_dim DH (64 or 32), fp16 operands.
//   scores[128x128] = Q K^T        2 x DH/16 wgmma m64n128k16 (query rows 0-63, 64-127), fp32 fragments -> smem score tile
//   P = exp(scale*(s - max)) masked  thread = query row, reads its score row; P held in registers, then -> smem (swizzled fp16)
//   out[128xDH] = P V              2 x 8 wgmma m64nDHk16, fragments -> smem
//   ctx[row, h*DH + :] = out / rowsum  (fp16: the A operand of the output projection)
// smem: one 68 KB region that holds, in turn, the Q and K tiles (16 KB each, TMA, 128B swizzle), the fp32 score tile, P
// (2 slabs x 16 KB) and the output tile; then V^T (2 slabs x 8 KB by TMA from the transposed buffer the QKV epilogue wrote).
// 85 KB per CTA: two CTAs share an SM, so one CTA's softmax overlaps the other's loads and MMAs.
// DH = 32 (MiniLM, BGE-small, E5-small: hidden 384 = 12 x 32) keeps every layout and descriptor of DH = 64.  The Q and K
// boxes still span 64 halves but start at column h*32, so they hold this head and its neighbour (TMA zero-fills past 2H for
// the last head) and QK^T issues only k-steps 0-1.  The V^T box still spans 64 rows from row (b*heads + h)*32; PV reads
// its first 32 rows (one 4 KB, 1 KB-aligned block of 8-row swizzle atoms per slab) as the N = 32 operand.  Attention is
// ~5% of such an encoder's flops, so the unused half of each box costs less than a second descriptor type would add.
// ------------------------------------------------------------------------------------------------
constexpr int ATT_THREADS = 128;
constexpr int ATT_S_LD = 128 + 4;                            // score tile row stride (floats): conflict-free row reads
constexpr int ATT_S_BYTES = 128 * ATT_S_LD * 4;
constexpr int ATT_REGION_BYTES = (ATT_S_BYTES + 1023) / 1024 * 1024;
// after the region: V^T 16 KB | the load barrier (64 B) | the score term's own bytes (Score::SMEM_BLOCK)
constexpr int ATT_OFF_VT = ATT_REGION_BYTES, ATT_OFF_BAR = ATT_OFF_VT + 16 * 1024, ATT_OFF_TERM = ATT_OFF_BAR + 64;
template <class Score>
constexpr int ATT_SMEM = ATT_OFF_TERM + Score::SMEM_BLOCK + 1024 /*align*/;

// S[128 x 128] = Q K^T for the query tile sQ and key tile sK (both [128 rows x 128 B], 128B swizzle) -> sS (fp32, ld ATT_S_LD).
// Issued by the whole warpgroup; returns once the products are in shared memory (the caller synchronises the CTA).
// Only the first DH halves of every row are the head's: DH / 16 k-steps.
template <int DH>
__device__ __forceinline__ void att_scores(const uint8_t *sQ, const uint8_t *sK, float *sS) {
    const uint64_t bd = wgmma_desc_sw128(smem_u32(sK));
#pragma unroll 1
    for (int half = 0; half < 2; ++half) {
        float s[64];
        const uint64_t a = wgmma_desc_sw128(smem_u32(sQ + half * 8192));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < DH / 16; ++k) wgmma_m64n128_f16(s, a + 2 * k, bd + 2 * k, k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_store_acc(s, sS + half * 64 * ATT_S_LD, ATT_S_LD);
    }
}
// O[128 x DH] (+)= P V with P = 2 slabs x [128 rows x 64 keys] and V^T = 2 slabs x [64 (d) x 64 keys] in shared memory,
// of which the first DH rows (d) are the head's
template <int DH>
__device__ __forceinline__ void att_pv(const uint8_t *sP, const uint8_t *sVt, float (&o)[2][DH / 2], bool accumulate) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        wgmma_fence();
#pragma unroll
        for (int slab = 0; slab < 2; ++slab) {
            const uint64_t a = wgmma_desc_sw128(smem_u32(sP + slab * 16384 + half * 8192));
            const uint64_t bd = wgmma_desc_sw128(smem_u32(sVt + slab * 8192));
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if constexpr (DH == 64) wgmma_m64n64_f16(o[half], a + 2 * k, bd + 2 * k, accumulate || (slab | k) != 0);
                else wgmma_m64n32_f16(o[half], a + 2 * k, bd + 2 * k, accumulate || (slab | k) != 0);
            }
        }
    }
    wgmma_commit();
    wgmma_wait<0>();
}
// P row qrow (32 keys from column c) as fp16 into the swizzled P slabs: slab (c / 64), 4 x 16-byte chunks
__device__ __forceinline__ void att_store_p(uint32_t sp_base, int qrow, int c, const uint32_t *pk) {
    const uint32_t prow = sp_base + (c >> 6) * 16384 + (qrow >> 3) * 1024 + (qrow & 7) * 128;
    const int ch0 = (c & 63) >> 3;
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) {
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(prow + (((ch0 + ch) ^ (qrow & 7)) << 4)),
                     "r"(pk[4 * ch]), "r"(pk[4 * ch + 1]), "r"(pk[4 * ch + 2]), "r"(pk[4 * ch + 3])
                     : "memory");
    }
}
// ctx[dst row, 0..DH-1] = fp16(out row * inv), out row read from the smem tile
template <int DH>
__device__ __forceinline__ void att_write_row(const float *orow, float inv, __half *dst) {
#pragma unroll
    for (int c = 0; c < DH; c += 8) {
        const float4 a = *reinterpret_cast<const float4 *>(orow + c);
        const float4 b = *reinterpret_cast<const float4 *>(orow + c + 4);
        __half2 h0 = __floats2half2_rn(a.x * inv, a.y * inv), h1 = __floats2half2_rn(a.z * inv, a.w * inv);
        __half2 h2 = __floats2half2_rn(b.x * inv, b.y * inv), h3 = __floats2half2_rn(b.z * inv, b.w * inv);
        uint4 pk;
        pk.x = *reinterpret_cast<uint32_t *>(&h0); pk.y = *reinterpret_cast<uint32_t *>(&h1);
        pk.z = *reinterpret_cast<uint32_t *>(&h2); pk.w = *reinterpret_cast<uint32_t *>(&h3);
        *reinterpret_cast<uint4 *>(dst + c) = pk;
    }
}

// sliding-window band of query q over keys [k0, k0 + 32): bit j set when |q - (k0 + j)| <= w; w = 0: no band (all set)
__device__ __forceinline__ uint32_t band_bits(int q, int k0, int w) {
    if (w <= 0) return 0xffffffffu;
    const int lo = q - w - k0, hi = q + w - k0;
    if (hi < 0 || lo > 31) return 0u;
    const uint32_t up = hi >= 31 ? 0xffffffffu : (2u << hi) - 1u;        // bits 0 .. hi
    const uint32_t dn = lo <= 0 ? 0xffffffffu : ~((1u << lo) - 1u);       // bits lo .. 31
    return up & dn;
}

// validity of keys [key0, key0 + 128) for query q (key < S, not padded, inside the band) as four 32-bit words held by
// every thread: lane l of a warp tests key key0 + 32 w + l once and ballots; the softmax loops only test bits
__device__ __forceinline__ void att_key_bits(const int32_t *mask, int64_t row0, int S, int key0, int q, int window, int lane,
                                             uint32_t (&kmask)[4]) {
#pragma unroll
    for (int w4 = 0; w4 < 4; ++w4) {
        const int key = key0 + 32 * w4 + lane;
        const bool ok = (key < S) && (!mask || mask[row0 + key] != 0);
        kmask[w4] = __ballot_sync(0xffffffffu, ok) & band_bits(q, key0 + 32 * w4, window);
    }
}
// P = exp2(r scale_log2 - mxs) of 32 scores (0 where the key bit is clear) as 16 fp16 pairs into pk; sum += their total
__device__ __forceinline__ void att_exp_pack(const float (&r)[32], uint32_t km, float scale_log2, float mxs, float &sum,
                                             uint32_t *pk) {
#pragma unroll
    for (int j = 0; j < 32; j += 2) {
        const float e0 = ((km >> j) & 1u) ? ex2_approx(fmaf(r[j], scale_log2, -mxs)) : 0.f;
        const float e1 = ((km >> (j + 1)) & 1u) ? ex2_approx(fmaf(r[j + 1], scale_log2, -mxs)) : 0.f;
        sum += e0 + e1;
        __half2 hh = __floats2half2_rn(e0, e1);
        pk[j >> 1] = *reinterpret_cast<uint32_t *>(&hh);
    }
}

// ---- score terms: what an encoder family adds to Q K^T before the softmax.  Both kernels take one as the `Score` template
// parameter and kernel argument, and call its hooks at fixed points; a hook a family does not need is empty.
// Where the calling CTA stands:
struct AttCta {
    uint8_t *smem;        // 1 KB-aligned base of the kernel's layout
    uint8_t *term;        // the score term's own bytes behind that layout (ATT_OFF_TERM / ATTS_OFF_TERM)
    int tid, h, heads;    // thread = query row of the block, head, heads of the encoder
    int q0, nblk;         // first query of the block, key blocks it visits from key 0 (attention_kernel: 0, 1)
};

// BERT, RoBERTa, DistilBERT, MiniLM (DH 32), ModernBERT: softmax(Q K^T / sqrt(DH) + mask), nothing added
struct ScorePlain {
    static constexpr int MIN_DH = 32;             // head dimensions the term is written for: MIN_DH .. 64
    static constexpr bool ONE_BLOCK = true;       // runs on attention_kernel as well as on attention_stream_kernel
    static constexpr int SCALE_TERMS = 1;         // logits are scores / sqrt(SCALE_TERMS DH)
    static constexpr bool EX2_ROWS = false;       // true: row() leaves ex2-domain logits, so the softmax scales by 1
    static constexpr int SMEM_BLOCK = 0, SMEM_STREAM = 0;   // own bytes in attention_kernel / attention_stream_kernel
    // the hooks, in call order.  init_barriers: thread 0, with the kernel's own barriers.  begin: every thread, once the
    // barriers are visible (first loads into the term's bytes).  add_block_terms / after_pv: every thread, visit i of the
    // streamed kernel, with the CTA synchronised after Q K^T reached the score tile / after P V retired (the P slabs are
    // free).  row: the 32 scores of the thread's row from key `key` on, after every read of them.
    __device__ __forceinline__ void init_barriers(const AttCta &) const {}
    __device__ __forceinline__ void begin(const AttCta &) const {}
    __device__ __forceinline__ void add_block_terms(const AttCta &, int) const {}
    __device__ __forceinline__ void row(float (&)[32], const AttCta &, int, float) const {}
    __device__ __forceinline__ void after_pv(const AttCta &, int) const {}
};

// MPNet relative position bias (modeling_mpnet.py MPNetEncoder.compute_position_bias), added to the scaled scores before
// the mask (window 0).  rel_bias row h holds the head's bias at entry (AC_ENCODER_MAX_S - 1) + key - q.  A CTA of queries
// q0 .. q0 + 127 and keys 0 .. 128 nblk - 1 stages entries from (AC_ENCODER_MAX_S - 128) - q0 on, times log2(e), so that
// query row qrow (q = q0 + qrow) finds the bias of key at sB[127 - qrow + key]: 32 lanes read 32 consecutive words,
// conflict-free.
struct ScoreRelBias : ScorePlain {
    const float *rel_bias;                        // [heads, 2 AC_ENCODER_MAX_S - 1]
    static constexpr int MIN_DH = 64;
    static constexpr bool EX2_ROWS = true;
    static constexpr int ATT_BIAS_OFS = AC_ENCODER_MAX_S - 128;
    // the staged entries: 255, and up to 128 (AC_ENCODER_MAX_S / 128) + 127
    static constexpr int SMEM_BLOCK = 1024, SMEM_STREAM = (AC_ENCODER_MAX_S + 128) * 4;
    __device__ __forceinline__ void begin(const AttCta &cta) const {
        const float *row = rel_bias + cta.h * (2 * AC_ENCODER_MAX_S - 1);
        float *sB = reinterpret_cast<float *>(cta.term);
        for (int t = cta.tid; t < 128 * cta.nblk + 127; t += ATT_THREADS)
            sB[t] = __ldg(row + ATT_BIAS_OFS - cta.q0 + t) * 1.44269504088896340736f;
    }
    // scores of 32 keys -> ex2-domain logits s scale log2(e) + bias log2(e)
    __device__ __forceinline__ void row(float (&r)[32], const AttCta &cta, int key, float scale_log2) const {
        const float *bq = reinterpret_cast<const float *>(cta.term) + 127 - cta.tid;
#pragma unroll
        for (int j = 0; j < 32; ++j) r[j] = fmaf(r[j], scale_log2, bq[key + j]);
    }
};

// window: ModernBERT sliding_attention half-window (keys |q - key| <= window), 0 = full attention.
template <int DH, class Score>
__global__ void __launch_bounds__(ATT_THREADS)
attention_kernel(const __grid_constant__ CUtensorMap tmap_qk, const __grid_constant__ CUtensorMap tmap_vt,
                 const int32_t *__restrict__ mask, int B, int S, int heads, int H, int window, __half *__restrict__ ctx,
                 const __grid_constant__ Score score) {
    static_assert(Score::ONE_BLOCK && DH >= Score::MIN_DH, "score term not written for this kernel or head dimension");
    static_assert(2 * (ATT_SMEM<Score> + 1024) <= 228 * 1024, "two attention CTAs must fit one SM");
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *sQ = smem;                    // [128 rows x 128 B]
    uint8_t *sK = smem + 16 * 1024;        // [128 rows x 128 B]
    float *sS = reinterpret_cast<float *>(smem);   // score tile, then output tile (after QK^T / PV retired)
    uint8_t *sP = smem;                    // 2 slabs x [128 rows x 128 B (64 keys)]   (after every score row was read)
    uint8_t *sVt = smem + ATT_OFF_VT;      // 2 slabs x [64 rows (d) x 128 B (64 keys)]
    uint64_t *bar_load = reinterpret_cast<uint64_t *>(smem + ATT_OFF_BAR);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int b = blockIdx.x / heads, h = blockIdx.x % heads;
    const int64_t row0 = static_cast<int64_t>(b) * S;
    const AttCta cta = {smem, smem + ATT_OFF_TERM, tid, h, heads, 0, 1};

    if (tid == 0) {
        tma_prefetch_desc(&tmap_qk);
        tma_prefetch_desc(&tmap_vt);
        mbar_init(bar_load, 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (tid == 0) {
        mbar_arrive_expect_tx(bar_load, 48 * 1024);
        const int r = static_cast<int>(row0);
        tma_load_2d(sQ, &tmap_qk, bar_load, h * DH, r);
        tma_load_2d(sK, &tmap_qk, bar_load, H + h * DH, r);
        const int vrow = (b * heads + h) * DH;                 // rows (b, h, d) of the transposed V buffer
        tma_load_2d(sVt, &tmap_vt, bar_load, 0, vrow);
        tma_load_2d(sVt + 8 * 1024, &tmap_vt, bar_load, 64, vrow);
    }
    score.begin(cta);
    // ---- S = Q K^T: both 64-row chains retire before the score tile overwrites Q and K
    mbar_wait_guarded(bar_load, 0);
    {
        float s0[64], s1[64];
        const uint64_t bd = wgmma_desc_sw128(smem_u32(sK));
        const uint64_t a0 = wgmma_desc_sw128(smem_u32(sQ)), a1 = wgmma_desc_sw128(smem_u32(sQ + 8192));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < DH / 16; ++k) wgmma_m64n128_f16(s0, a0 + 2 * k, bd + 2 * k, k != 0);
#pragma unroll
        for (int k = 0; k < DH / 16; ++k) wgmma_m64n128_f16(s1, a1 + 2 * k, bd + 2 * k, k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        __syncthreads();
        wgmma_store_acc(s0, sS, ATT_S_LD);
        wgmma_store_acc(s1, sS + 64 * ATT_S_LD, ATT_S_LD);
    }
    __syncthreads();

    // ---- softmax: thread = query row, two passes over the 128 score columns
    const int qrow = warp * 32 + lane;
    const float *srow = sS + qrow * ATT_S_LD;
    uint32_t kmask[4];
    att_key_bits(mask, row0, S, 0, qrow, window, lane, kmask);
    const float scale_log2 = rsqrtf(static_cast<float>(Score::SCALE_TERMS * DH)) * 1.44269504088896340736f;
    const float sl2 = Score::EX2_ROWS ? 1.f : scale_log2;
    float mx = -CUDART_INF_F;
#pragma unroll 1
    for (int c = 0; c < 128; c += 32) {
        float r[32];
        acc_row_ld32(srow + c, r);
        score.row(r, cta, c, scale_log2);
        const uint32_t km = c == 0 ? kmask[0] : c == 32 ? kmask[1] : c == 64 ? kmask[2] : kmask[3];
#pragma unroll
        for (int j = 0; j < 32; ++j)
            if ((km >> j) & 1u) mx = fmaxf(mx, r[j]);
    }
    float sum = 0.f;
    uint32_t pk[64];                       // the whole P row: P overwrites score rows other threads may still be reading
#pragma unroll
    for (int ci = 0; ci < 4; ++ci) {
        float r[32];
        acc_row_ld32(srow + 32 * ci, r);
        score.row(r, cta, 32 * ci, scale_log2);
        att_exp_pack(r, kmask[ci], sl2, mx * sl2, sum, pk + 16 * ci);
    }
    __syncthreads();                       // every score row has been read
    const uint32_t sp_base = smem_u32(sP);
#pragma unroll
    for (int ci = 0; ci < 4; ++ci) att_store_p(sp_base, qrow, 32 * ci, pk + 16 * ci);
    // generic-proxy smem writes (P) -> visible to the tensor-core (async) proxy
    fence_proxy_async_smem();
    __syncthreads();

    // ---- O = P V, staged over P once every warp's MMAs have read it
    float o[2][DH / 2];
    att_pv<DH>(sP, sVt, o, false);
    __syncthreads();
    wgmma_store_acc(o[0], sS, ATT_S_LD);
    wgmma_store_acc(o[1], sS + 64 * ATT_S_LD, ATT_S_LD);
    __syncthreads();
    const float inv = (sum > 0.f) ? 1.f / sum : 0.f;
    if (qrow < S) att_write_row<DH>(srow, inv, ctx + (row0 + qrow) * H + h * DH);
}

// ------------------------------------------------------------------------------------------------
// attention for 128 < S <= AC_MODERNBERT_MAX_S, head_dim 64 or 32: one CTA per (sequence, head, 128-query block), ONE
// pass over the key blocks with an online softmax.  BERT-family encoders pass window 0 and visit every key block.
//   key blocks    full layers visit all ceil(S / 128); sliding layers only those intersecting [q0 - w, q0 + 127 + w]
//                 (band_bits masks inside them), so a sliding layer costs O(S w) instead of O(S^2)
//   ring          K and V^T blocks come through two TMA stages: block i + 1 loads while block i runs its MMAs and softmax
//   softmax       thread = query row on the shared score tile: running row max m and row sum l; when m grows, the fp32
//                 O accumulator (wgmma registers) is scaled by exp(m_old - m_new), handed to the fragment rows
//                 16 warp + lane / 4 (+ 8, + 64) through shared memory.  A row that has seen no valid key yet (the ends of
//                 a sliding query block, holes in the mask) keeps m = -inf, P = 0 and a zero accumulator: the factor is
//                 0 there rather than exp((-inf) - (-inf))
//   P fp16, every accumulator fp32, as in the kernel above.  q_blocks = 1 (CLS-only tail next) computes rows 0..127 only.
// smem: Q 16 KB | K 2 x 16 KB | V^T 2 x 16 KB | P 32 KB | score tile 66 KB | factors 512 B | 2 barriers | the score term's
// own bytes (Score::SMEM_STREAM): one CTA per SM.
// ------------------------------------------------------------------------------------------------
constexpr int ATTS_STAGE_BYTES = 16 * 1024;
constexpr int ATTS_OFF_K = 16 * 1024, ATTS_OFF_VT = 48 * 1024, ATTS_OFF_P = 80 * 1024, ATTS_OFF_S = 112 * 1024;
constexpr int ATTS_OFF_BAR = ATTS_OFF_S + ATT_S_BYTES + 128 * 4, ATTS_OFF_TERM = ATTS_OFF_BAR + 2 * 8;
template <class Score>
constexpr int ATTS_SMEM = ATTS_OFF_TERM + Score::SMEM_STREAM + 1024 /*align*/;

// DeBERTa disentangled attention (modeling_deberta_v2.py DisentangledSelfAttention), on the streamed kernel only, which
// runs every DeBERTa sequence length (S <= 128 as one key block).  For query i and key j, r = i - j:
//     s(i, j) = (q_i . k_j + q_i . PosK[c(r)] + k_j . PosQ[c(r)]) / sqrt(3 dh)
// (HF gathers p2c at -bucket(j - i) + span, which is c(r) because the log bucket is odd).  In the tile of query block q0
// and key block k0, with a = i - q0, b = j - k0 and delta = q0 - k0, r = delta + a - b takes 255 values.  The ac_encoder
// holds, per (layer, delta, head), two fp16 boxes of 256 rows x 64 (ac_encoder::pos_g, built by pos_gather_kernel):
//     c2p  G[t] = PosK[c(delta + t - 127)]    C = Q G^T    (a, t) -> score (a, b = a - t + 127)
//     p2c  G[u] = PosQ[c(delta + 127 - u)]    C = K G^T    (b, u) -> score (a = b - u + 127, b)
// Each product is 2 x 2 wgmma m64n128k64 (query / key rows 0-63, 64-127 by G rows 0-127, 128-255) whose fragments are
// added straight into the fp32 score tile: every fragment element lands on at most one score and every score receives
// exactly one element per term, so a pass needs no atomics (the two passes are separated by a barrier).  Row 255 of a box
// is zero and never lands.  delta = 128 (blockIdx.y - key block); c(r) is monotone and saturates, so past some radius
// D every row of a box is the saturated one and the handle keeps only the boxes of blockIdx.y - key block in [-D, D]
// (n = 2 D + 1 of them, ac_encoder_create), a larger offset reading the box at +-D.  That bounds the boxes at any S.
// smem: the c2p box has its own 32 KB; the p2c box goes through the P slabs, free between PV and the next softmax.

// C = A G^T of one relative term over the 128 A rows (sA: Q or this key block's K) and the 256-row box sG, added into the
// score tile: c2p (P2C false) at (row, row - n + 127), p2c at (row - n + 127, row); n = the box row of the product column
template <bool P2C>
__device__ __forceinline__ void att_rel_term(const uint8_t *sA, const uint8_t *sG, float *sS) {
    const int t = threadIdx.x & 127;
    const int r0 = 16 * (t >> 5) + ((t & 31) >> 2), c0 = 2 * (t & 3);
#pragma unroll 1
    for (int half = 0; half < 2; ++half) {
#pragma unroll 1
        for (int nc = 0; nc < 2; ++nc) {
            float c[64];
            const uint64_t a = wgmma_desc_sw128(smem_u32(sA + half * 8192));
            const uint64_t bd = wgmma_desc_sw128(smem_u32(sG + nc * 16384));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_m64n128_f16(c, a + 2 * k, bd + 2 * k, k != 0);
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < 64; ++j) {
                const int row = 64 * half + r0 + 8 * ((j >> 1) & 1);
                const int other = row - (128 * nc + 8 * (j >> 2) + c0 + (j & 1)) + 127;
                if (other >= 0 && other < 128) {
                    float *dst = P2C ? sS + other * ATT_S_LD + row : sS + row * ATT_S_LD + other;
                    *dst += c[j];
                }
            }
        }
    }
}

struct ScoreDisent : ScorePlain {
    CUtensorMap tmap_pos;                         // 128-row boxes over ac_encoder::pos_g
    int pos_row0;                                 // first row of the layer's boxes
    int pos_d;                                    // D: the boxes cover block offsets -D .. D
    static constexpr int MIN_DH = 64;
    static constexpr bool ONE_BLOCK = false;
    static constexpr int SCALE_TERMS = 3;
    // own bytes: two barriers (the c2p box has landed, the p2c box has), then the c2p box at the layout's next 1 KB boundary
    static constexpr int OFF_G = (ATTS_OFF_TERM + 2 * 8 + 1023) / 1024 * 1024 - ATTS_OFF_TERM;
    static constexpr int SMEM_STREAM = OFF_G + 2 * ATTS_STAGE_BYTES;
    // the c2p (term 0) / p2c (term 1) box of visit i -> its own 32 KB / the P slabs; window 0, so visit i is key block i
    __device__ __forceinline__ void issue_pos(const AttCta &cta, int i, int term) const {
        const int d = min(max(static_cast<int>(blockIdx.y) - i, -pos_d), pos_d) + pos_d;
        const int row = pos_row0 + ((d * cta.heads + cta.h) * 2 + term) * 256;
        uint64_t *bar = reinterpret_cast<uint64_t *>(cta.term) + term;
        uint8_t *dst = term ? cta.smem + ATTS_OFF_P : cta.term + OFF_G;
        mbar_arrive_expect_tx(bar, 2 * ATTS_STAGE_BYTES);
        tma_load_2d(dst, &tmap_pos, bar, 0, row);
        tma_load_2d(dst + ATTS_STAGE_BYTES, &tmap_pos, bar, 0, row + 128);
    }
    __device__ __forceinline__ void init_barriers(const AttCta &cta) const {
        mbar_init(reinterpret_cast<uint64_t *>(cta.term), 1);
        mbar_init(reinterpret_cast<uint64_t *>(cta.term) + 1, 1);
    }
    __device__ __forceinline__ void begin(const AttCta &cta) const {
        if (cta.tid == 0) {
            issue_pos(cta, 0, 0);
            issue_pos(cta, 0, 1);
        }
    }
    __device__ __forceinline__ void add_block_terms(const AttCta &cta, int i) const {
        uint64_t *bar = reinterpret_cast<uint64_t *>(cta.term);
        float *sS = reinterpret_cast<float *>(cta.smem + ATTS_OFF_S);
        mbar_wait_guarded(bar, i & 1);
        att_rel_term<false>(cta.smem, cta.term + OFF_G, sS);
        __syncthreads();                                          // c2p added; its box is free
        if (cta.tid == 0 && i + 1 < cta.nblk) issue_pos(cta, i + 1, 0);
        mbar_wait_guarded(bar + 1, i & 1);
        att_rel_term<true>(cta.smem + ATTS_OFF_K + (i & 1) * ATTS_STAGE_BYTES, cta.smem + ATTS_OFF_P, sS);
        __syncthreads();                                          // p2c added; the P slabs are free
    }
    __device__ __forceinline__ void after_pv(const AttCta &cta, int i) const {
        if (cta.tid == 0 && i + 1 < cta.nblk) issue_pos(cta, i + 1, 1);
    }
};

template <int DH, class Score>
__global__ void __launch_bounds__(ATT_THREADS)
attention_stream_kernel(const __grid_constant__ CUtensorMap tmap_qk, const __grid_constant__ CUtensorMap tmap_vt,
                        const int32_t *__restrict__ mask, int B, int S, int heads, int H, int window, __half *__restrict__ ctx,
                        const __grid_constant__ Score score) {
    static_assert(DH >= Score::MIN_DH, "score term not written for this head dimension");
    static_assert(ATTS_SMEM<Score> <= 227 * 1024, "streamed attention CTA exceeds the shared-memory limit");
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *sQ = smem;                              // [128 x 128 B]
    uint8_t *sK = smem + ATTS_OFF_K;                 // stage st: [128 keys x 128 B]
    uint8_t *sVt = smem + ATTS_OFF_VT;               // stage st: 2 slabs x [64 (d) x 128 B (64 keys)]
    uint8_t *sP = smem + ATTS_OFF_P;                 // 2 slabs x [128 x 128 B (64 keys)]
    float *sS = reinterpret_cast<float *>(smem + ATTS_OFF_S);
    float *sAlpha = sS + 128 * ATT_S_LD;             // [128] rescale factor of each query row
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + ATTS_OFF_BAR);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int b = blockIdx.x / heads, h = blockIdx.x % heads;
    const int q0 = blockIdx.y * 128;
    const int64_t row0 = static_cast<int64_t>(b) * S;
    const int vrow = (b * heads + h) * DH;
    int kb0 = 0, kb1 = (S + 127) / 128;              // key blocks [kb0, kb1) of this query block
    if (window > 0) {
        kb0 = max(q0 - window, 0) / 128;
        kb1 = min(q0 + 127 + window, S - 1) / 128 + 1;
    }
    const int nblk = kb1 - kb0;
    const AttCta cta = {smem, smem + ATTS_OFF_TERM, tid, h, heads, q0, nblk};

    // visit i -> stage i & 1; the first visit also brings Q
    auto issue = [&](int i) {
        const int st = i & 1, key0 = (kb0 + i) * 128;
        mbar_arrive_expect_tx(bar + st, (i == 0 ? 3 : 2) * ATTS_STAGE_BYTES);
        if (i == 0) tma_load_2d(sQ, &tmap_qk, bar, h * DH, static_cast<int>(row0) + q0);
        tma_load_2d(sK + st * ATTS_STAGE_BYTES, &tmap_qk, bar + st, H + h * DH, static_cast<int>(row0) + key0);
        tma_load_2d(sVt + st * ATTS_STAGE_BYTES, &tmap_vt, bar + st, key0, vrow);
        tma_load_2d(sVt + st * ATTS_STAGE_BYTES + 8192, &tmap_vt, bar + st, key0 + 64, vrow);
    };
    if (tid == 0) {
        tma_prefetch_desc(&tmap_qk);
        tma_prefetch_desc(&tmap_vt);
        mbar_init(bar, 1);
        mbar_init(bar + 1, 1);
        score.init_barriers(cta);
        fence_mbar_init();
    }
    __syncthreads();
    if (tid == 0) {
        issue(0);
        if (nblk > 1) issue(1);
    }
    score.begin(cta);

    const int qrow = warp * 32 + lane;                            // row inside the query block
    const int qglob = q0 + qrow;                                  // position inside the sequence
    const float *srow = sS + qrow * ATT_S_LD;
    const float scale_log2 = rsqrtf(static_cast<float>(Score::SCALE_TERMS * DH)) * 1.44269504088896340736f;
    const float sl2 = Score::EX2_ROWS ? 1.f : scale_log2;
    const int frow = 16 * warp + (lane >> 2);                     // accumulator fragment rows frow, frow + 8 (+ 64)
    const uint32_t sp_base = smem_u32(sP);
    float mx = -CUDART_INF_F, sum = 0.f;
    float o[2][DH / 2];
#pragma unroll
    for (int half = 0; half < 2; ++half)
#pragma unroll
        for (int j = 0; j < DH / 2; ++j) o[half][j] = 0.f;

#pragma unroll 1
    for (int i = 0; i < nblk; ++i) {
        const int st = i & 1, key0 = (kb0 + i) * 128;
        mbar_wait_guarded(bar + st, (i >> 1) & 1);
        att_scores<DH>(sQ, sK + st * ATTS_STAGE_BYTES, sS);
        __syncthreads();
        score.add_block_terms(cta, i);

        uint32_t kmask[4];
        att_key_bits(mask, row0, S, key0, qglob, window, lane, kmask);
        float bmx = -CUDART_INF_F;
#pragma unroll
        for (int ci = 0; ci < 4; ++ci) {
            float r[32];
            acc_row_ld32(srow + 32 * ci, r);
            score.row(r, cta, key0 + 32 * ci, scale_log2);
#pragma unroll
            for (int jj = 0; jj < 32; ++jj)
                if ((kmask[ci] >> jj) & 1u) bmx = fmaxf(bmx, r[jj]);
        }
        const float mnew = fmaxf(mx, bmx);
        const float alpha = (mx == -CUDART_INF_F) ? 0.f : ex2_approx((mx - mnew) * sl2);
        const float mxs = (mnew == -CUDART_INF_F) ? 0.f : mnew * sl2;   // no valid key yet: every P below is 0
        float bsum = 0.f;
#pragma unroll
        for (int ci = 0; ci < 4; ++ci) {
            float r[32];
            acc_row_ld32(srow + 32 * ci, r);
            score.row(r, cta, key0 + 32 * ci, scale_log2);
            uint32_t pk[16];
            att_exp_pack(r, kmask[ci], sl2, mxs, bsum, pk);
            att_store_p(sp_base, qrow, 32 * ci, pk);
        }
        sum = fmaf(sum, alpha, bsum);
        mx = mnew;
        sAlpha[qrow] = alpha;
        fence_proxy_async_smem();
        __syncthreads();                                          // P and the factors are complete

#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const float a0 = sAlpha[64 * half + frow], a1 = sAlpha[64 * half + frow + 8];
#pragma unroll
            for (int j = 0; j < DH / 8; ++j) {
                o[half][4 * j] *= a0;
                o[half][4 * j + 1] *= a0;
                o[half][4 * j + 2] *= a1;
                o[half][4 * j + 3] *= a1;
            }
        }
        att_pv<DH>(sP, sVt + st * ATTS_STAGE_BYTES, o, true);
        __syncthreads();                                          // stage st, P, the score tile and the factors are free
        if (tid == 0 && i + 2 < nblk) issue(i + 2);
        score.after_pv(cta, i);
    }

    wgmma_store_acc(o[0], sS, ATT_S_LD);
    wgmma_store_acc(o[1], sS + 64 * ATT_S_LD, ATT_S_LD);
    __syncthreads();
    const float inv = (sum > 0.f) ? 1.f / sum : 0.f;
    if (qglob < S) att_write_row<DH>(srow, inv, ctx + (row0 + qglob) * H + h * DH);
}

// ------------------------------------------------------------------------------------------------
// long full attention: RoBERTa-arch encoders past AC_ENCODER_MAX_S (XLM-R: bge-m3, arctic-embed-l-v2.0), head_dim 64,
// window 0, no score term.  The contract of attention_stream_kernel<64, ScorePlain> (same arguments, grid, operand model
// and empty-row rule) with the softmax on the wgmma fragments.  One CTA of 288 threads per (sequence, head, 128-query block):
//   warp 8         producer: one lane TMA-loads Q once, then the K and V^T blocks of 128 keys through an ATTL_STAGES ring
//                  (full barriers: bytes landed; empty barriers: one arrival per consumer warp once its P V retired)
//   warpgroups 0-1 consumers, query rows 64 g .. 64 g + 63.  Per key block: S = Q K^T as 4 x wgmma m64n128k16 into 64 fp32
//                  registers; keys the mask or the sequence end exclude (one bit per key of the sequence, ballotted into
//                  shared memory once) become -inf; the row max and row sum reduce over the quad that holds a row
//                  (shfl_xor 1, 2); O is rescaled in registers; P is packed to f16x2 and is the REGISTER A operand of
//                  8 x wgmma m64n64k16 against the V^T slabs (the accumulator fragment of score columns [16 k, 16 k + 16) is
//                  the A fragment of k-step k)
// P is fp16, rounded against the running max; scores, the row sum (of the unrounded P, kept per thread and reduced once at
// the end) and O are fp32.  A row that has seen no valid key keeps m = -inf, P = 0 and the factor 0; its context is 0.
// Registers: 158 per thread with no spills (-Xptxas -v), so one CTA per SM; the two consumer warpgroups overlap each other's
// softmax with their MMAs.  smem: Q 16 KB | ATTL_STAGES x (K 16 KB | V^T 16 KB) | key bits (S / 8 B, <= 1 KB) | barriers.
// ------------------------------------------------------------------------------------------------
constexpr int ATTL_THREADS = 288;
constexpr int ATTL_STAGES = 4;
constexpr int ATTL_STAGE_BYTES = 32 * 1024;                    // K block | V^T block (2 slabs of 64 keys)
constexpr int ATTL_OFF_STAGE = 16 * 1024;
constexpr int ATTL_OFF_BITS = ATTL_OFF_STAGE + ATTL_STAGES * ATTL_STAGE_BYTES;
constexpr int ATTL_OFF_BAR = ATTL_OFF_BITS + AC_MODERNBERT_MAX_S / 8;
constexpr int ATTL_SMEM = ATTL_OFF_BAR + (1 + 2 * ATTL_STAGES) * 8 + 1024 /*align*/;
static_assert(ATTL_SMEM <= 227 * 1024, "long-attention CTA exceeds the shared-memory limit");

__global__ void __launch_bounds__(ATTL_THREADS, 1)
attention_long_kernel(const __grid_constant__ CUtensorMap tmap_qk, const __grid_constant__ CUtensorMap tmap_vt,
                      const int32_t *__restrict__ mask, int B, int S, int heads, int H, int /*window: 0*/,
                      __half *__restrict__ ctx, const __grid_constant__ ScorePlain) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *sQ = smem;                                                // [128 x 128 B]: rows 64 g .. for warpgroup g
    uint32_t *sBits = reinterpret_cast<uint32_t *>(smem + ATTL_OFF_BITS);   // bit j of word w: key 32 w + j is attended
    uint64_t *bar_q = reinterpret_cast<uint64_t *>(smem + ATTL_OFF_BAR);
    uint64_t *full = bar_q + 1, *empty = full + ATTL_STAGES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int b = blockIdx.x / heads, h = blockIdx.x % heads;
    const int q0 = blockIdx.y * 128;
    const int row0 = b * S;
    const int nblk = (S + 127) / 128;

    if (tid == 0) {
        tma_prefetch_desc(&tmap_qk);
        tma_prefetch_desc(&tmap_vt);
        mbar_init(bar_q, 1);
        for (int st = 0; st < ATTL_STAGES; ++st) {
            mbar_init(full + st, 1);
            mbar_init(empty + st, 8);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            const int vrow = (b * heads + h) * 64;
            mbar_arrive_expect_tx(bar_q, 16 * 1024);
            tma_load_2d(sQ, &tmap_qk, bar_q, h * 64, row0 + q0);
            for (int i = 0; i < nblk; ++i) {
                const int st = i % ATTL_STAGES, key0 = i * 128;
                if (i >= ATTL_STAGES) mbar_wait_guarded(empty + st, (i / ATTL_STAGES - 1) & 1);
                uint8_t *sK = smem + ATTL_OFF_STAGE + st * ATTL_STAGE_BYTES, *sVt = sK + 16 * 1024;
                mbar_arrive_expect_tx(full + st, ATTL_STAGE_BYTES);
                tma_load_2d(sK, &tmap_qk, full + st, H + h * 64, row0 + key0);
                tma_load_2d(sVt, &tmap_vt, full + st, key0, vrow);
                tma_load_2d(sVt + 8192, &tmap_vt, full + st, key0 + 64, vrow);
            }
        }
        return;
    }

    // ---- consumers: the key bits of every key block (keys past S are clear), then the key blocks
    for (int w = warp; w < 4 * nblk; w += 8) {
        const int key = 32 * w + lane;
        const bool ok = key < S && (!mask || mask[row0 + key] != 0);
        const uint32_t bits = __ballot_sync(0xffffffffu, ok);
        if (lane == 0) sBits[w] = bits;
    }
    named_bar_sync(1, 256);

    const int g = warp >> 2;
    const int r0 = 16 * (warp & 3) + (lane >> 2), c2 = 2 * (lane & 3);   // fragment rows r0, r0 + 8; columns 8 j + c2 (+1)
    const float sl2 = 0.125f * 1.44269504088896340736f;                 // log2(e) / sqrt(64)
    float o[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) o[j] = 0.f;
    float mx0 = -CUDART_INF_F, mx1 = -CUDART_INF_F, sum0 = 0.f, sum1 = 0.f;
    const uint64_t qa = wgmma_desc_sw128(smem_u32(sQ + g * 8192));
    mbar_wait_guarded(bar_q, 0);

#pragma unroll 1
    for (int i = 0; i < nblk; ++i) {
        const int st = i % ATTL_STAGES;
        const uint8_t *sK = smem + ATTL_OFF_STAGE + st * ATTL_STAGE_BYTES, *sVt = sK + 16 * 1024;
        mbar_wait_guarded(full + st, (i / ATTL_STAGES) & 1);
        float s[64];
        {
            const uint64_t bd = wgmma_desc_sw128(smem_u32(sK));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_m64n128_f16(s, qa + 2 * k, bd + 2 * k, k != 0);
            wgmma_commit();
            wgmma_wait<0>();
        }
        const uint4 kw = *reinterpret_cast<const uint4 *>(sBits + 4 * i);
        if ((kw.x & kw.y & kw.z & kw.w) != 0xffffffffu) {
            const uint32_t words[4] = {kw.x, kw.y, kw.z, kw.w};
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const uint32_t bits = words[j >> 2] >> (8 * (j & 3) + c2);
                if (!(bits & 1u)) s[4 * j] = s[4 * j + 2] = -CUDART_INF_F;
                if (!(bits & 2u)) s[4 * j + 1] = s[4 * j + 3] = -CUDART_INF_F;
            }
        }
        float m0 = mx0, m1 = mx1;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            m0 = fmaxf(m0, fmaxf(s[4 * j], s[4 * j + 1]));
            m1 = fmaxf(m1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
        }
#pragma unroll
        for (int x = 1; x <= 2; x <<= 1) {
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, x));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, x));
        }
        const float alpha0 = (mx0 == -CUDART_INF_F) ? 0.f : ex2_approx((mx0 - m0) * sl2);
        const float alpha1 = (mx1 == -CUDART_INF_F) ? 0.f : ex2_approx((mx1 - m1) * sl2);
        const float ms0 = (m0 == -CUDART_INF_F) ? 0.f : m0 * sl2;      // no valid key yet: every P below is 0
        const float ms1 = (m1 == -CUDART_INF_F) ? 0.f : m1 * sl2;
        mx0 = m0;
        mx1 = m1;
        uint32_t p[32];
        float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float e0 = ex2_approx(fmaf(s[4 * j], sl2, -ms0)), e1 = ex2_approx(fmaf(s[4 * j + 1], sl2, -ms0));
            const float e2 = ex2_approx(fmaf(s[4 * j + 2], sl2, -ms1)), e3 = ex2_approx(fmaf(s[4 * j + 3], sl2, -ms1));
            ps0 += e0 + e1;
            ps1 += e2 + e3;
            __half2 h01 = __floats2half2_rn(e0, e1), h23 = __floats2half2_rn(e2, e3);
            p[2 * j] = *reinterpret_cast<uint32_t *>(&h01);
            p[2 * j + 1] = *reinterpret_cast<uint32_t *>(&h23);
        }
        sum0 = fmaf(sum0, alpha0, ps0);
        sum1 = fmaf(sum1, alpha1, ps1);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[4 * j] *= alpha0;
            o[4 * j + 1] *= alpha0;
            o[4 * j + 2] *= alpha1;
            o[4 * j + 3] *= alpha1;
        }
        {
            const uint64_t bv = wgmma_desc_sw128(smem_u32(sVt));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t a[4] = {p[4 * k], p[4 * k + 1], p[4 * k + 2], p[4 * k + 3]};
                wgmma_m64n64_f16_rs(o, a, bv + (k >> 2) * 512 + 2 * (k & 3), 1u);   // slab k / 4 is 8192 B on
            }
            wgmma_commit();
            wgmma_wait<0>();
        }
        if (lane == 0) mbar_arrive(empty + st);
    }

#pragma unroll
    for (int x = 1; x <= 2; x <<= 1) {
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, x);
        sum1 += __shfl_xor_sync(0xffffffffu, sum1, x);
    }
    const float inv0 = (sum0 > 0.f) ? 1.f / sum0 : 0.f, inv1 = (sum1 > 0.f) ? 1.f / sum1 : 0.f;
    const int q = q0 + 64 * g + r0;
    __half *dst = ctx + (static_cast<int64_t>(row0) + q) * H + h * 64 + c2;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (q < S) *reinterpret_cast<__half2 *>(dst + 8 * j) = __floats2half2_rn(o[4 * j] * inv0, o[4 * j + 1] * inv0);
        if (q + 8 < S)
            *reinterpret_cast<__half2 *>(dst + 8 * static_cast<int64_t>(H) + 8 * j) =
                __floats2half2_rn(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1);
    }
}

// last layer, deferred flow: CLS rows of the attention context and of LN_pending(y) (two-pass statistics from the fp32 sums)
__global__ void gather_cls_ln_kernel(const __half *__restrict__ ctx, const float *__restrict__ y, int B, int S, int H,
                                     const float *__restrict__ g, const float *__restrict__ b, float eps,
                                     __half *__restrict__ ctx_cls, float *__restrict__ x_cls) {
    const int bq = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (bq >= B) return;
    const int64_t src = static_cast<int64_t>(bq) * S * H, dst = static_cast<int64_t>(bq) * H;
    for (int i = lane; i < H / 8; i += 32)
        reinterpret_cast<uint4 *>(ctx_cls + dst)[i] = reinterpret_cast<const uint4 *>(ctx + src)[i];
    const int nv = H / 128;
    float4 x[LN_MAXV];
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i)
        if (i < nv) x[i] = *reinterpret_cast<const float4 *>(y + src + (lane + 32 * i) * 4);
    ln_row(x, nv, H, g, b, eps, lane, x_cls + dst, nullptr);
}

// DeBERTa operand boxes of attention_stream_kernel<64, ScoreDisent> (see att_rel_term): row ((((l n + d) heads + h) 2 + term)
// 256 + t) = fp16 (RNE) of PosK (term 0) / PosQ (term 1) [l, c(r), 64 h .. 64 h + 63] with delta = 128 (d - n / 2),
// r = delta + t - 127 (c2p) or delta + 127 - t (p2c), c(r) = rel_index[radius - 1 + r]; row t = 255 is zero.  rel_index
// covers |r| < radius; a box row past it (|r| >= radius: no query-key pair of an accepted S) reads the nearest entry.
// pos_key / pos_query [layers, 2 span, H] fp32.  64 threads per row, 4 rows per block.
__global__ void pos_gather_kernel(const float *__restrict__ pos_key, const float *__restrict__ pos_query,
                                  const int32_t *__restrict__ rel_index, int radius, int n, int span, int heads, int H,
                                  __half *__restrict__ out) {
    const int64_t row = static_cast<int64_t>(blockIdx.x) * 4 + (threadIdx.x >> 6);
    const int col = threadIdx.x & 63;
    const int t = static_cast<int>(row % 256), term = static_cast<int>((row / 256) % 2);
    const int h = static_cast<int>((row / 512) % heads);
    const int64_t ld = row / (512 * static_cast<int64_t>(heads));          // l n + d
    const int d = static_cast<int>(ld % n);
    const int64_t l = ld / n;
    float v = 0.f;
    if (t < 255) {
        const int delta = 128 * (d - n / 2);
        const int r = min(max(term ? delta + 127 - t : delta + t - 127, 1 - radius), radius - 1);
        const int c = min(max(rel_index[radius - 1 + r], 0), 2 * span - 1);
        v = (term ? pos_query : pos_key)[(l * 2 * span + c) * H + 64 * h + col];
    }
    out[row * 64 + col] = __float2half_rn(v);
}

}  // namespace ac

// ================================================================================================
// encoder handle
// ================================================================================================
using namespace ac;

// One encoder layer, fields by role; where BERT-family (post-LN) and ModernBERT (pre-LN) layers differ, the comment says so.
struct Layer {
    // fp16 GEMM operands with their GEMM_BLOCK_N-row-box maps: QKV [3H, H] and FFN1 (BERT W1 [I, H], ModernBERT Wi [2I, H]
    // interleaved for GeGLU) consume un-normalised residual sums and are packed as fp16(gamma * W) by pack_consumer
    __half *wqkv = nullptr, *wo = nullptr, *w1 = nullptr, *w2 = nullptr;
    CUtensorMap m_wqkv, m_wo, m_w1, m_w2;
    // rank-1 corrections of the deferred-LayerNorm consumers: c1 (row sums of the packed weight), c0 (W beta + bias)
    float *c1qkv = nullptr, *c0qkv = nullptr, *c1f = nullptr, *c0f = nullptr;
    float *bo = nullptr, *b2 = nullptr;   // residual biases of Wo / W2 (ModernBERT: zeros)
    // LayerNorm FFN1 consumes: BERT attention.output.LayerNorm (left pending on the residual sums), ModernBERT mlp_norm
    // (beta zeros; the residual sums stay raw)
    float *ln_ffn_w = nullptr, *ln_ffn_b = nullptr;
    // LayerNorm of the layer output: BERT output.LayerNorm (left pending on the residual sums), ModernBERT final_norm (beta
    // zeros) in the last layer only (the next layer's attn_norm is folded into its Wqkv)
    float *ln_out_w = nullptr, *ln_out_b = nullptr;
    int window = 0;                       // sliding-attention half-window, 0 = full attention (always 0 for BERT)
};

struct ac_encoder {
    ac_encoder_config cfg;
    // packed weights (device): fp16 GEMM operands, fp32 everything else.  ModernBERT: no pos / type, emb_ln_b = zeros
    float *word = nullptr, *pos = nullptr, *type = nullptr, *emb_ln_w = nullptr, *emb_ln_b = nullptr;
    // embedding projection [H, E] (fp16) and its bias, NULL without one; m_emb views e->ctx as the [T, E] LayerNorm-ed
    // embedding rows it consumes (ctx is free until layer 0's attention)
    __half *emb_proj_w = nullptr;
    float *emb_proj_b = nullptr;
    CUtensorMap m_emb, m_emb_proj;
    std::vector<Layer> layers;
    __half *w1_last = nullptr;            // plain fp16 FFN1 weight of the last layer (CLS-only tail runs on materialised LayerNorm rows)
    float *b1_last = nullptr;             // its bias (ModernBERT: zeros)
    // activations: fp32 residual sums x (+ tmp for a materialised final LayerNorm); fp16 GEMM operands xh, qk, vT, ctx, ffn
    float *x = nullptr, *tmp = nullptr;
    __half *xh = nullptr, *qk = nullptr, *vT = nullptr, *ctx = nullptr, *ffn = nullptr;
    size_t T = 0;           // token capacity (multiple of 128)
    size_t vt_elems = 0;
    // compact CLS-row buffers of the last layer (Bc rows)
    size_t Bc = 0;
    float *x_cls = nullptr, *tmp_cls = nullptr;
    __half *xh_cls = nullptr, *ctx_cls = nullptr, *ffn_cls = nullptr;
    CUtensorMap m_xh_cls, m_ctx_cls, m_ffn_cls;
    // cached TMA descriptors: A operands (128-row boxes) and weights (128-row boxes = the B half one CTA of a pair stages)
    CUtensorMap m_xh, m_ctx, m_ffn, m_qk_att, m_vt_att;
    int vt_B = -1, vt_S = -1;
    CUtensorMap p_w1_last;
    // row statistics (ping-pong) and the per-GEMM_EPI_COLS-column partials the residual epilogues write
    float2 *stats_a = nullptr, *stats_b = nullptr, *stats_id = nullptr, *parts = nullptr;
    float *ones = nullptr, *zeros = nullptr;   // ones [H]; zeros [max(3H, 2I)]: beta / bias of the bias-free ModernBERT
    float *rope[2] = {nullptr, nullptr};       // RoPE tables [max_pos, 64]: ModernBERT (full, sliding layers), rotary (full)
    float *rel_bias = nullptr;                 // MPNet relative position bias [heads, 2 AC_ENCODER_MAX_S - 1]; NULL otherwise
    // DeBERTa c2p / p2c operand boxes [layers, 2 pos_d + 1, heads, 2 (c2p, p2c), 256, 64] fp16 (pos_gather_kernel) and
    // their 128-row-box map; NULL otherwise
    __half *pos_g = nullptr;
    CUtensorMap m_pos;
    int pos_d = 0;                        // the boxes' block offsets -pos_d .. pos_d (deberta_box_radius)
    std::vector<void *> allocs;
    int last_B = 0, last_S = 0;           // shape of the previous forward; its full hidden state (cls_only = 0) is in tmp
    bool last_cls_only = false;
};

static int launch_cls_normalize(const float *x, int B, int S, int H, float *out, cudaStream_t s) {
    const int wpb = 8;
    cls_normalize_kernel<<<(B + wpb - 1) / wpb, wpb * 32, 0, s>>>(x, B, S, H, out);
    AC_LAUNCH_CHECK();
    return AC_OK;
}

// Every attention variant the library runs, with the dynamic shared memory the kernel is allowed and launched with and its
// block size (rows in the enum's order).  All take the same arguments up to their score term.
struct AttVariant { const void *kernel; int smem, threads; };
enum { ATT_PLAIN64, ATT_PLAIN32, ATT_RELBIAS, ATTS_PLAIN64, ATTS_PLAIN32, ATTS_RELBIAS, ATTS_DISENT, ATTL_PLAIN64, ATT_VARIANTS };
static const AttVariant att_variants[ATT_VARIANTS] = {
    {reinterpret_cast<const void *>(attention_kernel<64, ScorePlain>), ATT_SMEM<ScorePlain>, ATT_THREADS},
    {reinterpret_cast<const void *>(attention_kernel<32, ScorePlain>), ATT_SMEM<ScorePlain>, ATT_THREADS},
    {reinterpret_cast<const void *>(attention_kernel<64, ScoreRelBias>), ATT_SMEM<ScoreRelBias>, ATT_THREADS},
    {reinterpret_cast<const void *>(attention_stream_kernel<64, ScorePlain>), ATTS_SMEM<ScorePlain>, ATT_THREADS},
    {reinterpret_cast<const void *>(attention_stream_kernel<32, ScorePlain>), ATTS_SMEM<ScorePlain>, ATT_THREADS},
    {reinterpret_cast<const void *>(attention_stream_kernel<64, ScoreRelBias>), ATTS_SMEM<ScoreRelBias>, ATT_THREADS},
    {reinterpret_cast<const void *>(attention_stream_kernel<64, ScoreDisent>), ATTS_SMEM<ScoreDisent>, ATT_THREADS},
    {reinterpret_cast<const void *>(attention_long_kernel), ATTL_SMEM, ATTL_THREADS},
};

// softmax(Q K^T / sqrt(head_dim) [+ MPNet relative bias] + mask) V out of e->qk / e->vT into e->ctx; window = sliding
// half-window, 0 = full attention.  S <= 128 runs attention_kernel, longer sequences attention_stream_kernel over 128-query
// blocks; DeBERTa runs attention_stream_kernel<64, ScoreDisent> at every length, with layer `layer`'s c2p / p2c boxes.
// Past AC_ENCODER_MAX_S every encoder but ModernBERT and DeBERTa (in practice RoBERTa-arch ones with a long position table,
// check_shape_map_vt) runs attention_long_kernel; ModernBERT keeps attention_stream_kernel at every length.
// cls_rows: only row 0 of every sequence is read afterwards (the CLS-only tail), so only the first query block is computed.
static int launch_attention(ac_encoder *e, const int32_t *mask, int B, int S, int window, bool cls_rows, int layer,
                            cudaStream_t s) {
    const ac_encoder_config &c = e->cfg;
    int H = c.hidden, heads = c.heads;
    const int dh = H / heads;                 // 64 or 32 (ac_encoder_create); 64 with a relative bias or DeBERTa's boxes
    AC_REQUIRE(S <= AC_ENCODER_MAX_S || dh == 64, "attention: S=%d > %d needs head_dim 64 (ModernBERT)", S, AC_ENCODER_MAX_S);
    // per-device: the attribute is a property of the (function, device) pair
    static bool att_attr[64] = {};
    int dev = 0;
    AC_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !att_attr[dev]) {
        for (const AttVariant &v : att_variants)
            AC_CUDA(cudaFuncSetAttribute(v.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, v.smem));
        if (dev >= 0 && dev < 64) att_attr[dev] = true;
    }
    // algorithmic flops over the keys each computed query attends to at the true sequence length (the 128-wide tiles do
    // more): (2w + 1) clipped to [0, S) in sliding layers
    const int q_blocks = cls_rows ? 1 : (S + 127) / 128;
    const int nq = std::min(S, 128 * q_blocks);
    double keys = 0.0;
    if (window > 0) {
        for (int q = 0; q < nq; ++q) keys += std::min(S - 1, q + window) - std::max(0, q - window) + 1;
    } else {
        keys = static_cast<double>(nq) * S;
    }
    const int slot = prof_begin(PROF_ATTENTION, 4.0 * B * c.heads * keys * dh, 0.0, s);
    const bool streamed = e->pos_g || S > 128;
    ScorePlain plain;
    ScoreRelBias bias;
    ScoreDisent disent;
    void *score = &plain;
    int id = dh == 32 ? (streamed ? ATTS_PLAIN32 : ATT_PLAIN32) : (streamed ? ATTS_PLAIN64 : ATT_PLAIN64);
    if (e->pos_g) {
        disent.tmap_pos = e->m_pos;
        disent.pos_row0 = layer * (2 * e->pos_d + 1) * heads * 2 * 256;
        disent.pos_d = e->pos_d;
        score = &disent;
        id = ATTS_DISENT;
    } else if (e->rel_bias) {
        bias.rel_bias = e->rel_bias;
        score = &bias;
        id = streamed ? ATTS_RELBIAS : ATT_RELBIAS;
    } else if (S > AC_ENCODER_MAX_S && c.arch != AC_ARCH_MODERNBERT) {
        id = ATTL_PLAIN64;                    // head_dim 64 (checked above), window 0 (only ModernBERT has bands)
    }
    const AttVariant &v = att_variants[id];
    void *args[] = {&e->m_qk_att, &e->m_vt_att, &mask, &B, &S, &heads, &H, &window, &e->ctx, score};
    // a launch error is the runtime's last error, which AC_LAUNCH_CHECK reads
    cudaLaunchKernel(v.kernel, dim3(B * heads, streamed ? q_blocks : 1), dim3(v.threads), args, v.smem, s);
    prof_end(slot, s);
    AC_LAUNCH_CHECK();
    return AC_OK;
}

template <class T>
static int dev_alloc(ac_encoder *e, T **p, size_t elems) {
    void *q = nullptr;
    AC_CUDA(cudaMalloc(&q, elems * sizeof(T)));
    e->allocs.push_back(q);
    *p = static_cast<T *>(q);
    return AC_OK;
}

static int pack_f32(ac_encoder *e, float **dst, const float *src, size_t n) {
    int rc = dev_alloc(e, dst, n);
    if (rc) return rc;
    round_copy_kernel<<<256, 256>>>(src, *dst, static_cast<int64_t>(n), 0);
    AC_LAUNCH_CHECK();
    return AC_OK;
}
static int pack_f16(ac_encoder *e, __half **dst, const float *src, size_t n) {
    int rc = dev_alloc(e, dst, n);
    if (rc) return rc;
    to_half_kernel<<<256, 256>>>(src, *dst, static_cast<int64_t>(n));
    AC_LAUNCH_CHECK();
    return AC_OK;
}

extern "C" int ac_encoder_destroy(ac_encoder *enc) {
    if (!enc) return AC_OK;
    for (void *p : enc->allocs) cudaFree(p);
    delete enc;
    return AC_OK;
}

// Packs a deferred-LayerNorm consumer of sums pending LayerNorm (gamma, beta), NULL = identity: the n weights W[j] [N, K]
// with biases bias[j] (bias NULL: none) stacked into one operand *wp [n N, K] and its vectors *c1, *c0 [n N].
// glu != 0: W is a GeGLU weight (input rows, then gate rows), see pack_defer_kernel.
static int pack_consumer(ac_encoder *e, int n, const float *const *W, const float *const *bias, const float *gamma,
                         const float *beta, int N, int K, int glu, __half **wp, float **c1, float **c0) {
    const size_t NK = static_cast<size_t>(N) * K;
    int rc;
    if ((rc = dev_alloc(e, wp, n * NK)) || (rc = dev_alloc(e, c1, static_cast<size_t>(n) * N)) ||
        (rc = dev_alloc(e, c0, static_cast<size_t>(n) * N)))
        return rc;
    for (int j = 0; j < n; ++j) {
        pack_defer_kernel<<<(N + 7) / 8, 256>>>(W[j], bias ? bias[j] : nullptr, gamma, beta, N, K, *wp + j * NK, *c1 + j * N,
                                                *c0 + j * N, glu);
        if ((rc = check_cuda(cudaGetLastError(), "pack_defer_kernel"))) return rc;
    }
    return AC_OK;
}

// D of a DeBERTa handle's operand boxes, from its index table idx (entry radius - 1 + r = c(r), |r| < radius): the least d
// for which c is constant for r >= 128 d - 127 and for r <= 127 - 128 d, so that the boxes at +-d, and every box farther
// out, hold one row throughout (pos_gather_kernel) and a larger block offset may read the box at +-d.  At most
// (radius - 1) / 128, the largest block offset of a sequence of S <= radius.  Published v3 settings give 5.
static int deberta_box_radius(const std::vector<int32_t> &idx, int radius) {
    const int cap = (radius - 1) / 128;
    const auto c = [&](int r) { return idx[radius - 1 + r]; };
    const auto saturated = [&](int d) {
        for (int r = 128 * d - 127; r < radius; ++r)
            if (c(r) != c(radius - 1)) return false;
        for (int r = 127 - 128 * d; r > -radius; --r)
            if (c(r) != c(1 - radius)) return false;
        return true;
    };
    int d = 0;
    while (d < cap && !saturated(d)) ++d;
    return d;
}

extern "C" int ac_encoder_create(const ac_encoder_config *cfg, const ac_encoder_weights *w, ac_encoder **out) {
    AC_REQUIRE(cfg && w && out, "ac_encoder_create: null argument");
    const bool mb = cfg->arch == AC_ARCH_MODERNBERT;
    AC_REQUIRE(!mb || (cfg->max_pos >= AC_ENCODER_MAX_S && cfg->max_pos <= AC_MODERNBERT_MAX_S && cfg->layer_sliding &&
                       cfg->sliding_window > 0 && cfg->rope_full && cfg->rope_sliding && w->wqkv && w->wi && w->final_norm_w &&
                       (cfg->layers == 1 || w->attn_norm_w)),
               "ac_encoder_create: ModernBERT needs %d <= max_pos <= %d (max_pos=%d), layer_sliding, sliding_window > 0, both "
               "RoPE tables, wqkv, wi, final_norm_w and attn_norm_w", AC_ENCODER_MAX_S, AC_MODERNBERT_MAX_S, cfg->max_pos);
    const bool rot = cfg->arch == AC_ARCH_ROTARY;
    AC_REQUIRE(!rot || (cfg->rope_full && cfg->max_pos >= AC_ENCODER_MAX_S && cfg->max_pos <= AC_MODERNBERT_MAX_S),
               "ac_encoder_create: AC_ARCH_ROTARY needs rope_full and %d <= max_pos <= %d (max_pos=%d)", AC_ENCODER_MAX_S,
               AC_MODERNBERT_MAX_S, cfg->max_pos);
    const bool eb = cfg->arch == AC_ARCH_EUROBERT;
    AC_REQUIRE(!eb || (cfg->rope_full && cfg->max_pos >= AC_ENCODER_MAX_S && cfg->max_pos <= AC_MODERNBERT_MAX_S),
               "ac_encoder_create: AC_ARCH_EUROBERT needs rope_full and %d <= max_pos <= %d (max_pos=%d)", AC_ENCODER_MAX_S,
               AC_MODERNBERT_MAX_S, cfg->max_pos);
    AC_REQUIRE(!eb || (w->wqkv && w->wi && w->attn_norm_w && w->final_norm_w),
               "ac_encoder_create: AC_ARCH_EUROBERT needs wqkv, wi, attn_norm_w (every layer's, layer 0's included) and "
               "final_norm_w");
    AC_REQUIRE(cfg->precision == AC_PREC_F16, "ac_encoder_create: only AC_PREC_F16 (fp16 operands, fp32 accumulate) is implemented");
    AC_REQUIRE(cfg->hidden % 128 == 0 && cfg->hidden <= 1024, "ac_encoder_create: hidden=%d must be a multiple of 128, <= 1024", cfg->hidden);
    // the attention kernels take head_dim 64 or 32; the RoPE epilogue pairs (d, d + 32) inside a 64-column head
    AC_REQUIRE(cfg->heads > 0 && cfg->hidden % cfg->heads == 0 &&
                   (cfg->hidden / cfg->heads == 64 || (!mb && !rot && !eb && cfg->hidden / cfg->heads == 32)),
               "ac_encoder_create: head_dim must be %s (hidden=%d heads=%d)",
               mb ? "64 for ModernBERT" : rot ? "64 for AC_ARCH_ROTARY" : eb ? "64 for AC_ARCH_EUROBERT" : "64 or 32",
               cfg->hidden, cfg->heads);
    const bool mp = cfg->arch == AC_ARCH_MPNET;
    AC_REQUIRE(!mp || (cfg->rel_bias && cfg->hidden == 64 * cfg->heads),
               "ac_encoder_create: MPNet needs rel_bias and head_dim 64 (hidden=%d heads=%d)", cfg->hidden, cfg->heads);
    const bool db = cfg->arch == AC_ARCH_DEBERTA;
    AC_REQUIRE(!db || (cfg->pos_key && cfg->pos_query && cfg->rel_index && cfg->pos_span > 0 &&
                       cfg->hidden == 64 * cfg->heads),
               "ac_encoder_create: DeBERTa needs pos_key, pos_query, rel_index, pos_span > 0 (pos_span=%d) and head_dim 64 "
               "(hidden=%d heads=%d)", cfg->pos_span, cfg->hidden, cfg->heads);
    AC_REQUIRE(cfg->rel_radius == 0 ||
                   (db && cfg->rel_radius > AC_ENCODER_MAX_S && cfg->rel_radius <= AC_MODERNBERT_MAX_S),
               "ac_encoder_create: rel_radius=%d must be 0 (AC_ENCODER_MAX_S), or %d < rel_radius <= %d on an "
               "AC_ARCH_DEBERTA encoder (arch=%d)", cfg->rel_radius, AC_ENCODER_MAX_S, AC_MODERNBERT_MAX_S, cfg->arch);
    AC_REQUIRE(cfg->intermediate % 64 == 0 && cfg->layers > 0 && cfg->max_tokens > 0, "ac_encoder_create: bad dims");
    AC_REQUIRE(cfg->ffn_act == AC_FFN_GELU_ERF || cfg->ffn_act == AC_FFN_GELU_TANH || cfg->ffn_act == AC_FFN_SWIGLU,
               "ac_encoder_create: unknown ffn_act=%d", cfg->ffn_act);
    const bool swiglu = cfg->ffn_act == AC_FFN_SWIGLU;
    AC_REQUIRE(!swiglu || rot || eb,
               "ac_encoder_create: ffn_act=%d (AC_FFN_SWIGLU) is implemented for AC_ARCH_ROTARY / AC_ARCH_EUROBERT only (arch=%d)",
               cfg->ffn_act, cfg->arch);
    AC_REQUIRE(!eb || swiglu, "ac_encoder_create: AC_ARCH_EUROBERT takes ffn_act=%d (AC_FFN_SWIGLU) only (ffn_act=%d)",
               AC_FFN_SWIGLU, cfg->ffn_act);
    const int E = cfg->embedding_size ? cfg->embedding_size : cfg->hidden;
    AC_REQUIRE(!mb || cfg->ffn_act == AC_FFN_GELU_ERF, "ac_encoder_create: ModernBERT takes no ffn_act=%d (its FFN is GeGLU)",
               cfg->ffn_act);
    // the projection runs after the embedding LayerNorm (ALBERT, ELECTRA); DeBERTa-v2's embed_proj runs before it
    AC_REQUIRE(!w->emb_proj_w || cfg->arch == AC_ARCH_BERT || cfg->arch == AC_ARCH_ROBERTA,
               "ac_encoder_create: an embedding projection (emb_proj_w) is implemented for AC_ARCH_BERT / AC_ARCH_ROBERTA "
               "only (arch=%d)", cfg->arch);
    AC_REQUIRE(w->emb_proj_w ? (w->emb_proj_b && E > 0 && E % 128 == 0 && E <= cfg->hidden) : E == cfg->hidden,
               "ac_encoder_create: embedding_size=%d (hidden=%d) with%s emb_proj_w: a projection needs emb_proj_b and a "
               "width that is a multiple of 128 and <= hidden; without one embedding_size must be 0 or hidden",
               cfg->embedding_size, cfg->hidden, w->emb_proj_w ? "" : "out");
    int rc = ac_device_check();
    if (rc) return rc;
    ac_encoder *e = new ac_encoder();
    e->cfg = *cfg;
    e->cfg.embedding_size = E;        // 0 resolved to hidden: forward_layers reads the width from here
    const int H = cfg->hidden, I = cfg->intermediate, L = cfg->layers;
    const int n1 = (mb || swiglu) ? 2 * I : I;   // rows of the first FFN weight (GLU: activated rows + multiplier rows)
    const size_t T = static_cast<size_t>((cfg->max_tokens + 127) / 128 * 128);
    e->T = T;
#define TRY(x) do { rc = (x); if (rc) { ac_encoder_destroy(e); return rc; } } while (0)
    e->cfg.layer_sliding = nullptr;   // copied into e->layers / e->rope below
    e->cfg.rope_full = e->cfg.rope_sliding = nullptr;
    e->cfg.rel_bias = nullptr;        // copied into e->rel_bias below
    e->cfg.pos_key = e->cfg.pos_query = nullptr;   // gathered into e->pos_g below
    e->cfg.rel_index = nullptr;
    // ones / zeros are filled with the other constants after packing; the bias-free ModernBERT roles point at zeros
    const int nzeros = std::max(3 * H, 2 * I);
    TRY(dev_alloc(e, &e->ones, H));
    TRY(dev_alloc(e, &e->zeros, nzeros));
    e->layers.resize(L);
    const size_t HH = static_cast<size_t>(H) * H, HI = static_cast<size_t>(H) * I;
    if (mb || eb) {
        // ModernBERT (modeling_modernbert.py): no biases or LayerNorm betas.  Wqkv consumes the sums pending attn_norm
        // (Identity in layer 0), Wi the sums pending mlp_norm.
        // EuroBERT (modeling_eurobert.py) the same pre-norm block with RMSNorms: no embedding norm, so layer 0's Wqkv
        // consumes the raw embeddings pending input_layernorm (attn_norm_w[0]); full attention in every layer; Wi is
        // cat(gate_proj, up_proj), the same interleaved row order for SwiGLU
        Layer &last = e->layers[L - 1];
        TRY(pack_f32(e, &e->word, w->word_emb, static_cast<size_t>(cfg->vocab) * H));
        if (mb) TRY(pack_f32(e, &e->emb_ln_w, w->emb_ln_w, H));
        TRY(pack_f32(e, &last.ln_out_w, w->final_norm_w, H));
        TRY(pack_f32(e, &e->rope[0], cfg->rope_full, static_cast<size_t>(cfg->max_pos) * 64));
        if (mb) TRY(pack_f32(e, &e->rope[1], cfg->rope_sliding, static_cast<size_t>(cfg->max_pos) * 64));
        e->emb_ln_b = e->b1_last = last.ln_out_b = e->zeros;
        for (int l = 0; l < L; ++l) {
            Layer &ly = e->layers[l];
            ly.window = mb && cfg->layer_sliding[l] ? cfg->sliding_window : 0;
            ly.bo = ly.b2 = ly.ln_ffn_b = e->zeros;
            TRY(pack_consumer(e, 1, &w->wqkv[l], nullptr, (l || eb) ? w->attn_norm_w[l] : nullptr, nullptr, 3 * H, H, 0,
                              &ly.wqkv, &ly.c1qkv, &ly.c0qkv));
            TRY(pack_f16(e, &ly.wo, w->ao_w[l], HH));
            TRY(pack_f32(e, &ly.ln_ffn_w, w->ao_ln_w[l], H));
            TRY(pack_consumer(e, 1, &w->wi[l], nullptr, w->ao_ln_w[l], nullptr, 2 * I, H, 1, &ly.w1, &ly.c1f, &ly.c0f));
            TRY(pack_f16(e, &ly.w2, w->ff2_w[l], HI));
        }
        if (cfg->cls_only) {
            // plain interleaved Wi of the last layer: the CLS-only tail materialises mlp_norm (c1 / c0 are not used)
            float *c1, *c0;
            TRY(pack_consumer(e, 1, &w->wi[L - 1], nullptr, nullptr, nullptr, 2 * I, H, 1, &e->w1_last, &c1, &c0));
        }
    } else {
        TRY(pack_f32(e, &e->word, w->word_emb, static_cast<size_t>(cfg->vocab) * E));
        if (rot) {
            // no position table: RoPE on q and k (table rope[0]); the embedding kernel reads one zero row (forward_layers)
            e->pos = e->zeros;
            TRY(pack_f32(e, &e->rope[0], cfg->rope_full, static_cast<size_t>(cfg->max_pos) * 64));
        } else {
            TRY(pack_f32(e, &e->pos, w->pos_emb, static_cast<size_t>(cfg->max_pos) * E));
        }
        TRY(pack_f32(e, &e->type, w->type_emb, static_cast<size_t>(cfg->type_vocab) * E));
        TRY(pack_f32(e, &e->emb_ln_w, w->emb_ln_w, E));
        TRY(pack_f32(e, &e->emb_ln_b, w->emb_ln_b, E));
        if (w->emb_proj_w) {
            TRY(pack_f16(e, &e->emb_proj_w, w->emb_proj_w, static_cast<size_t>(H) * E));
            TRY(pack_f32(e, &e->emb_proj_b, w->emb_proj_b, H));
        }
        if (mp) TRY(pack_f32(e, &e->rel_bias, cfg->rel_bias, static_cast<size_t>(cfg->heads) * (2 * AC_ENCODER_MAX_S - 1)));
        if (db) {
            const int R = e->cfg.rel_radius = cfg->rel_radius ? cfg->rel_radius : AC_ENCODER_MAX_S;
            if (R > AC_ENCODER_MAX_S) {
                // past max_pos the embedding kernel re-reads the table's last row: only a table of zeros (no absolute
                // positions, position_biased_input = False) is position-free
                std::vector<float> pos(static_cast<size_t>(cfg->max_pos) * E);
                TRY(check_cuda(cudaMemcpy(pos.data(), e->pos, pos.size() * sizeof(float), cudaMemcpyDeviceToHost),
                               "copy pos_emb"));
                if (std::any_of(pos.begin(), pos.end(), [](float v) { return v != 0.f; })) {
                    set_error("ac_encoder_create: rel_radius=%d needs an all-zero pos_emb (a DeBERTa encoder without "
                              "absolute positions, position_biased_input = False)", R);
                    ac_encoder_destroy(e);
                    return AC_E_INVALID;
                }
            }
            std::vector<int32_t> idx(2 * R - 1);
            TRY(check_cuda(cudaMemcpy(idx.data(), cfg->rel_index, idx.size() * sizeof(int32_t), cudaMemcpyDeviceToHost),
                           "copy rel_index"));
            e->pos_d = deberta_box_radius(idx, R);
            const int n = 2 * e->pos_d + 1;
            const size_t rows = static_cast<size_t>(L) * n * cfg->heads * 2 * 256;
            TRY(dev_alloc(e, &e->pos_g, rows * 64));
            pos_gather_kernel<<<static_cast<unsigned>(rows / 4), 256>>>(cfg->pos_key, cfg->pos_query, cfg->rel_index, R, n,
                                                                        cfg->pos_span, cfg->heads, H, e->pos_g);
            TRY(check_cuda(cudaGetLastError(), "pos_gather_kernel"));
            TRY(make_tmap_2d(&e->m_pos, e->pos_g, 2, rows, 64, 128, 128, 64));
        }
        // Shared packing: a packed operand whose sources (weights, biases and the LayerNorm folded into it) are the very
        // pointers of an earlier layer's is that layer's buffers.  ALBERT's cross-layer sharing thus packs one set of weights
        // plus a second QKV (layer 0's consumes the embeddings, the others the sums pending full_layer_layer_norm).
        using Src = std::array<const float *, 8>;
        const auto qkv_src = [&](int l) {
            return Src{w->q_w[l], w->k_w[l], w->v_w[l], w->q_b[l], w->k_b[l], w->v_b[l], l ? w->out_ln_w[l - 1] : nullptr,
                       l ? w->out_ln_b[l - 1] : nullptr};
        };
        const auto ffn1_src = [&](int l) { return Src{w->ff1_w[l], w->ff1_b[l], w->ao_ln_w[l], w->ao_ln_b[l]}; };
        const auto earlier = [&](int l, const auto &src) {    // first layer j < l with the same sources, or -1
            for (int j = 0; j < l; ++j)
                if (src(j) == src(l)) return j;
            return -1;
        };
        // a single-source operand: fp32 copy (bias, LayerNorm) or fp16 copy (plain weight) of src[l], or layer j's
        const auto copy_of = [&](auto Layer::*field, const float *const *src, int l, size_t n) -> int {
            const int j = earlier(l, [&](int i) { return Src{src[i]}; });
            if (j >= 0) {
                e->layers[l].*field = e->layers[j].*field;
                return AC_OK;
            }
            if constexpr (std::is_same_v<decltype(e->layers[l].*field), __half *&>)
                return pack_f16(e, &(e->layers[l].*field), src[l], n);
            else
                return pack_f32(e, &(e->layers[l].*field), src[l], n);
        };
        for (int l = 0; l < L; ++l) {
            Layer &ly = e->layers[l];
            // the fused QKV [3H, H] of layer l consumes the sums pending the output LayerNorm of layer l-1 (identity for
            // layer 0: the embeddings arrive normalised, or un-normalised from the projection), FFN1 the sums pending the
            // attention-output LayerNorm of layer l
            if (const int j = earlier(l, qkv_src); j >= 0) {
                ly.wqkv = e->layers[j].wqkv, ly.c1qkv = e->layers[j].c1qkv, ly.c0qkv = e->layers[j].c0qkv;
            } else {
                const float *ws[3] = {w->q_w[l], w->k_w[l], w->v_w[l]};
                const float *bs[3] = {w->q_b[l], w->k_b[l], w->v_b[l]};
                TRY(pack_consumer(e, 3, ws, bs, l ? w->out_ln_w[l - 1] : nullptr, l ? w->out_ln_b[l - 1] : nullptr, H, H, 0,
                                  &ly.wqkv, &ly.c1qkv, &ly.c0qkv));
            }
            TRY(copy_of(&Layer::wo, w->ao_w, l, HH));
            TRY(copy_of(&Layer::bo, w->ao_b, l, H));
            TRY(copy_of(&Layer::ln_ffn_w, w->ao_ln_w, l, H));
            TRY(copy_of(&Layer::ln_ffn_b, w->ao_ln_b, l, H));
            if (const int j = earlier(l, ffn1_src); j >= 0) {
                ly.w1 = e->layers[j].w1, ly.c1f = e->layers[j].c1f, ly.c0f = e->layers[j].c0f;
            } else {
                TRY(pack_consumer(e, 1, &w->ff1_w[l], &w->ff1_b[l], w->ao_ln_w[l], w->ao_ln_b[l], n1, H, swiglu, &ly.w1,
                                  &ly.c1f, &ly.c0f));
            }
            TRY(copy_of(&Layer::w2, w->ff2_w, l, HI));
            TRY(copy_of(&Layer::b2, w->ff2_b, l, H));
            TRY(copy_of(&Layer::ln_out_w, w->out_ln_w, l, H));
            TRY(copy_of(&Layer::ln_out_b, w->out_ln_b, l, H));
        }
        if (cfg->cls_only && swiglu) {
            // plain interleaved FFN1 of the last layer and its interleaved bias (c0 with no LayerNorm folded in)
            float *c1;
            TRY(pack_consumer(e, 1, &w->ff1_w[L - 1], &w->ff1_b[L - 1], nullptr, nullptr, n1, H, 1, &e->w1_last, &c1,
                              &e->b1_last));
        } else if (cfg->cls_only) {
            TRY(pack_f16(e, &e->w1_last, w->ff1_w[L - 1], HI));
            TRY(pack_f32(e, &e->b1_last, w->ff1_b[L - 1], I));
        }
    }
    TRY(dev_alloc(e, &e->stats_a, T));
    TRY(dev_alloc(e, &e->stats_b, T));
    TRY(dev_alloc(e, &e->stats_id, T));
    TRY(dev_alloc(e, &e->parts, static_cast<size_t>(H / GEMM_EPI_COLS) * T));
    fill_stats_identity_kernel<<<static_cast<unsigned>((T + 255) / 256), 256>>>(e->stats_id, static_cast<int64_t>(T));
    fill_value_kernel<<<(H + 255) / 256, 256>>>(e->ones, H, 1.f);
    fill_value_kernel<<<(nzeros + 255) / 256, 256>>>(e->zeros, nzeros, 0.f);
    TRY(check_cuda(cudaGetLastError(), "deferred-LayerNorm constants"));
    e->vt_elems = 2 * T * H;     // (b, h, d) rows x S_pad keys, S_pad = roundup(S, 8) <= 2*S for S >= 8
    TRY(dev_alloc(e, &e->x, T * H));
    TRY(dev_alloc(e, &e->tmp, T * H));
    TRY(dev_alloc(e, &e->xh, T * H));
    TRY(dev_alloc(e, &e->qk, T * 2 * H));
    TRY(dev_alloc(e, &e->vT, e->vt_elems));
    TRY(dev_alloc(e, &e->ctx, T * H));
    TRY(dev_alloc(e, &e->ffn, T * I));
    e->Bc = T < 16384 ? T : 16384;
    TRY(dev_alloc(e, &e->x_cls, e->Bc * H));
    TRY(dev_alloc(e, &e->tmp_cls, e->Bc * H));
    TRY(dev_alloc(e, &e->xh_cls, e->Bc * H));
    TRY(dev_alloc(e, &e->ctx_cls, e->Bc * H));
    TRY(dev_alloc(e, &e->ffn_cls, e->Bc * I));
    TRY(check_cuda(cudaMemset(e->xh_cls, 0, e->Bc * H * sizeof(__half)), "memset xh_cls"));
    TRY(check_cuda(cudaMemset(e->ctx_cls, 0, e->Bc * H * sizeof(__half)), "memset ctx_cls"));
    TRY(check_cuda(cudaMemset(e->ffn_cls, 0, e->Bc * I * sizeof(__half)), "memset ffn_cls"));
    TRY(check_cuda(cudaMemset(e->qk, 0, T * 2 * H * sizeof(__half)), "memset qk"));
    TRY(check_cuda(cudaMemset(e->vT, 0, e->vt_elems * sizeof(__half)), "memset vT"));
    TRY(check_cuda(cudaMemset(e->xh, 0, T * H * sizeof(__half)), "memset xh"));
    TRY(check_cuda(cudaMemset(e->ctx, 0, T * H * sizeof(__half)), "memset ctx"));
    TRY(check_cuda(cudaMemset(e->ffn, 0, T * I * sizeof(__half)), "memset ffn"));
    // TMA descriptors (fp16: 64 elements = 128 bytes per box row)
    TRY(make_tmap_2d(&e->m_xh, e->xh, 2, T, H, static_cast<uint64_t>(H) * 2, GEMM_BLOCK_M, 64));
    TRY(make_tmap_2d(&e->m_ctx, e->ctx, 2, T, H, static_cast<uint64_t>(H) * 2, GEMM_BLOCK_M, 64));
    TRY(make_tmap_2d(&e->m_ffn, e->ffn, 2, T, I, static_cast<uint64_t>(I) * 2, GEMM_BLOCK_M, 64));
    TRY(make_tmap_2d(&e->m_qk_att, e->qk, 2, T, 2 * H, static_cast<uint64_t>(2 * H) * 2, 128, 64));
    TRY(make_tmap_2d(&e->m_xh_cls, e->xh_cls, 2, e->Bc, H, static_cast<uint64_t>(H) * 2, GEMM_BLOCK_M, 64));
    TRY(make_tmap_2d(&e->m_ctx_cls, e->ctx_cls, 2, e->Bc, H, static_cast<uint64_t>(H) * 2, GEMM_BLOCK_M, 64));
    TRY(make_tmap_2d(&e->m_ffn_cls, e->ffn_cls, 2, e->Bc, I, static_cast<uint64_t>(I) * 2, GEMM_BLOCK_M, 64));
    if (e->emb_proj_w) {
        TRY(make_tmap_2d(&e->m_emb, e->ctx, 2, T, E, static_cast<uint64_t>(E) * 2, GEMM_BLOCK_M, 64));
        TRY(make_tmap_2d(&e->m_emb_proj, e->emb_proj_w, 2, H, E, static_cast<uint64_t>(E) * 2, GEMM_BLOCK_N, 64));
    }
    for (Layer &ly : e->layers) {
        TRY(make_tmap_2d(&ly.m_wqkv, ly.wqkv, 2, 3 * H, H, static_cast<uint64_t>(H) * 2, GEMM_BLOCK_N, 64));
        TRY(make_tmap_2d(&ly.m_wo, ly.wo, 2, H, H, static_cast<uint64_t>(H) * 2, GEMM_BLOCK_N, 64));
        TRY(make_tmap_2d(&ly.m_w1, ly.w1, 2, n1, H, static_cast<uint64_t>(H) * 2, GEMM_BLOCK_N, 64));
        TRY(make_tmap_2d(&ly.m_w2, ly.w2, 2, H, I, static_cast<uint64_t>(I) * 2, GEMM_BLOCK_N, 64));
    }
    if (cfg->cls_only) TRY(make_tmap_2d(&e->p_w1_last, e->w1_last, 2, n1, H, static_cast<uint64_t>(H) * 2, GEMM_BLOCK_N, 64));
    TRY(check_cuda(cudaDeviceSynchronize(), "encoder_create sync"));
#undef TRY
    *out = e;
    return AC_OK;
}

// One encoder projection = one GEMM (gemm_tc.cuh).  tb is the weight's GEMM_BLOCK_N-row-box map.
template <class Epi>
static int launch_linear(const CUtensorMap &ta, const CUtensorMap &tb, int M, int N, int K, const Epi &epi, cudaStream_t s) {
    return launch_gemm_tc<Epi, false, GEMM_KIND_F16>(ta, tb, M, N, K, epi, s);
}

// ---- one function per projection role: forward_layers and the parity entry ac_encoder_projection both run these, so the
// epilogue, operand maps, biases, tables and pending LayerNorm of a role are stated once.  M = B * S rows.

// ALBERT / ELECTRA embedding projection: e->ctx (LayerNorm-ed embedding rows, width E) -> e->x, e->xh
static int run_emb_proj(ac_encoder *e, int M, cudaStream_t s) {
    const int H = e->cfg.hidden;
    EpiEmbProj ep{.bias = e->emb_proj_b, .y = e->x, .yh = e->xh, .M = M, .N = H, .ld = H};
    return launch_linear(e->m_emb, e->m_emb_proj, M, H, e->cfg.embedding_size, ep, s);
}

// fused QKV of layer l on e->xh with the consumed norm's row statistics `stats` -> q | k in e->qk (RoPE with the layer's
// table: the sliding one in a ModernBERT sliding layer), V^T in e->vT
template <bool ROPE>
static int run_qkv(ac_encoder *e, int l, int B, int S, const float2 *stats, cudaStream_t s) {
    const int H = e->cfg.hidden, M = B * S;
    const Layer &ly = e->layers[l];
    EpiQKV<ROPE> eq{.qk = {.bias = ly.c0qkv, .c1 = ly.c1qkv, .row_stats = stats, .Y = e->qk, .M = M, .N = 3 * H, .ldy = 2 * H,
                           .S = S, .rope = e->rope[ly.window ? 1 : 0]},
                    .vT = e->vT, .vt_col0 = 2 * H, .S_pad = (S + 7) / 8 * 8, .H = H};
    return launch_linear(e->m_xh, ly.m_wqkv, M, 3 * H, H, eq, s);
}

// The LayerNorm pending on the residual sums when layer l's Wo (ffn = false) or W2 (ffn = true) adds them back, with the
// sums' statistics `stats`: post-LN blocks leave the previous layer's output LayerNorm (nothing before layer 0) and the
// layer's attention-output LayerNorm pending; pre-LN blocks keep the identity pending throughout.
struct PendingNorm { const float2 *stats; const float *gamma, *beta; };
template <bool PRE_LN>
static PendingNorm pending_norm(const ac_encoder *e, int l, bool ffn, const float2 *stats) {
    if (PRE_LN || (!ffn && l == 0)) return {e->stats_id, e->ones, e->zeros};
    if (ffn) return {stats, e->layers[l].ln_ffn_w, e->layers[l].ln_ffn_b};
    return {stats, e->layers[l - 1].ln_out_w, e->layers[l - 1].ln_out_b};
}

// residual projection of layer l, Wo on e->ctx (ffn = false) or W2 on e->ffn (ffn = true), in place on e->x / e->xh:
// y <- a W^T + b + LN_pending(y), then the row statistics of the new sums into stats_out
template <bool PRE_LN, Norm NORM>
static int run_resid(ac_encoder *e, int l, bool ffn, int M, const float2 *stats, float2 *stats_out, cudaStream_t s) {
    const ac_encoder_config &c = e->cfg;
    const int H = c.hidden;
    const int64_t pstride = static_cast<int64_t>(e->T);
    const Layer &ly = e->layers[l];
    const PendingNorm p = pending_norm<PRE_LN>(e, l, ffn, stats);
    EpiResidDefer ep{.bias = ffn ? ly.b2 : ly.bo, .y = e->x, .yh = e->xh, .stats_prev = p.stats, .gamma = p.gamma, .beta = p.beta,
                     .parts = e->parts, .part_stride = pstride, .M = M, .N = H, .ld = H};
    int rc = launch_linear(ffn ? e->m_ffn : e->m_ctx, ffn ? ly.m_w2 : ly.m_wo, M, H, ffn ? c.intermediate : H, ep, s);
    if (rc) return rc;
    ln_stats_kernel<NORM><<<(M + 255) / 256, 256, 0, s>>>(e->parts, H / GEMM_EPI_COLS, pstride, M, H, c.ln_eps, stats_out);
    AC_LAUNCH_CHECK();
    return AC_OK;
}

// accumulator columns of FFN1 (GLU: activated + multiplier rows)
template <Act FFN_ACT>
static int ffn1_cols(const ac_encoder *e) {
    return FFN_ACT == Act::GeGLU || FFN_ACT == Act::SwiGLU ? 2 * e->cfg.intermediate : e->cfg.intermediate;
}

// FFN1 of layer l on e->xh, consuming its pending norm with row statistics `stats` -> e->ffn
template <Act FFN_ACT>
static int run_ffn1(ac_encoder *e, int l, int M, const float2 *stats, cudaStream_t s) {
    const Layer &ly = e->layers[l];
    EpiF16<FFN_ACT, true> e1{.bias = ly.c0f, .c1 = ly.c1f, .row_stats = stats, .Y = e->ffn, .M = M, .N = ffn1_cols<FFN_ACT>(e),
                             .ldy = e->cfg.intermediate};
    return launch_linear(e->m_xh, ly.m_w1, M, e1.N, e->cfg.hidden, e1, s);
}

// FFN1 of the last layer on materialised LayerNorm rows (the CLS-only tail): the plain weight w1_last on `ta` -> out
template <Act FFN_ACT>
static int run_ffn1_rows(ac_encoder *e, const CUtensorMap &ta, __half *out, int M, cudaStream_t s) {
    EpiF16<FFN_ACT, false> e1{.bias = e->b1_last, .Y = out, .M = M, .N = ffn1_cols<FFN_ACT>(e), .ldy = e->cfg.intermediate};
    return launch_linear(ta, e->p_w1_last, M, e1.N, e->cfg.hidden, e1, s);
}

// The layer stack, for post-LN (BERT / RoBERTa / DistilBERT, modeling_bert.py) or pre-LN (ModernBERT,
// modeling_modernbert.py ModernBertModel.forward; EuroBERT, modeling_eurobert.py, with RMSNorm and SwiGLU) blocks:
//     post-LN   y = LN1(y + attn(y))               y = LN2(y + GELU-FFN(y))               out = y
//     pre-LN    y = y + attn(attn_norm(y))         y = y + GeGLU-FFN(mlp_norm(y))         out = final_norm(y)
// e->x holds the un-normalised residual sums y, e->xh their fp16 copy.  QKV and FFN1 apply the LayerNorm they consume
// deferred; the residual epilogues add LN_pending(y), carried as (row statistics, gamma, beta).  That pending LayerNorm is
// the one decision the block kinds differ in: post-LN blocks leave LN1 / LN2 pending, pre-LN blocks keep the identity
// (stats (0, 1), gamma 1, beta 0) pending throughout.  The rest is the epilogue type (RoPE, GeGLU) and data in e->layers.
// ROPE: q and k rotated in the QKV epilogue (ModernBERT, EuroBERT; post-LN AC_ARCH_ROTARY, which has no position table).
// FFN_ACT: GeGLU (ModernBERT), SwiGLU (EuroBERT), or the post-LN encoder's (ac_encoder_config.ffn_act: exact-erf or tanh
// GELU, SwiGLU).
// NORM: RMSNorm for EuroBERT's pre-norm block (input_layernorm, post_attention_layernorm, norm).  Its residual stream starts
// as the raw embedding rows, so layer 0's QKV consumes them with their RMS statistics instead of the identity.
template <bool PRE_LN, bool ROPE, Act FFN_ACT, Norm NORM>
static int forward_layers(ac_encoder *e, const int32_t *ids, const int32_t *mask, const int32_t *type_ids, int B, int S,
                          float *out_unit_cls, cudaStream_t s) {
    static_assert(PRE_LN ? ROPE && FFN_ACT == (NORM == Norm::Layer ? Act::GeGLU : Act::SwiGLU)
                         : NORM == Norm::Layer && FFN_ACT != Act::GeGLU,
                  "pre-LN blocks are ModernBERT's (LayerNorm, RoPE, GeGLU) and EuroBERT's (RMSNorm, RoPE, SwiGLU); post-LN "
                  "blocks use LayerNorm");
    const ac_encoder_config &c = e->cfg;
    const int H = c.hidden, I = c.intermediate, M = B * S;
    // a post-LN RoPE encoder's e->pos is one zero row: the embedding kernel's clamp to max_pos - 1 = 0 reads it
    const int emb_pos = (ROPE && !PRE_LN) ? 1 : c.max_pos;
    const int wpb = 8;
    const int row_blocks = (M + wpb - 1) / wpb;
    const bool cls_tail = c.cls_only && static_cast<size_t>(B) <= e->Bc;
    int rc;
    // the embeddings arrive normalised (or projected): identity statistics for layer 0's QKV (and the identity LayerNorm
    // pending, pending_norm); EuroBERT's arrive raw, with the RMS statistics of layer 0's input_layernorm in stats_a
    const float2 *st_qkv = e->stats_id;
    if constexpr (NORM == Norm::Rms) {
        embed_ln_kernel<true, true><<<row_blocks, wpb * 32, 0, s>>>(ids, nullptr, e->word, nullptr, nullptr, nullptr, nullptr,
                                                                    c.ln_eps, B, S, H, c.arch, c.pad_idx, c.vocab, c.max_pos,
                                                                    c.type_vocab, e->x, e->xh, e->stats_a);
        AC_LAUNCH_CHECK();
        st_qkv = e->stats_a;
    } else if (!e->emb_proj_w) {
        embed_ln_kernel<true><<<row_blocks, wpb * 32, 0, s>>>(ids, PRE_LN ? nullptr : type_ids, e->word, e->pos, e->type,
                                                              e->emb_ln_w, e->emb_ln_b, c.ln_eps, B, S, H, c.arch, c.pad_idx,
                                                              c.vocab, emb_pos, c.type_vocab, e->x, e->xh);
        AC_LAUNCH_CHECK();
    } else {
        // factorized embeddings: LayerNorm at width E into the ctx scratch (fp16), then y = LN(emb) Wp^T + bp at width H
        const int E = c.embedding_size;
        embed_ln_kernel<false><<<row_blocks, wpb * 32, 0, s>>>(ids, type_ids, e->word, e->pos, e->type, e->emb_ln_w,
                                                               e->emb_ln_b, c.ln_eps, B, S, E, c.arch, c.pad_idx, c.vocab,
                                                               c.max_pos, c.type_vocab, nullptr, e->ctx);
        AC_LAUNCH_CHECK();
        if ((rc = run_emb_proj(e, M, s))) return rc;
    }
    for (int l = 0; l < c.layers; ++l) {
        const Layer &ly = e->layers[l];
        if ((rc = run_qkv<ROPE>(e, l, B, S, st_qkv, s))) return rc;
        if ((rc = launch_attention(e, mask, B, S, ly.window, l == c.layers - 1 && cls_tail, l, s))) return rc;
        if (l == c.layers - 1 && cls_tail) break;
        // attention output projection + residual: y <- ctx Wo^T + bo + LN_pending(y); statistics of the new sums
        if ((rc = run_resid<PRE_LN, NORM>(e, l, false, M, e->stats_a, e->stats_b, s))) return rc;
        if ((rc = run_ffn1<FFN_ACT>(e, l, M, e->stats_b, s))) return rc;
        // FFN output projection + residual: y <- ffn W2^T + b2 + LN_pending(y)
        if ((rc = run_resid<PRE_LN, NORM>(e, l, true, M, e->stats_b, e->stats_a, s))) return rc;
        st_qkv = e->stats_a;
    }
    const Layer &last = e->layers.back();
    if (cls_tail) {
        // ---- CLS-only tail of the last layer (classifier.py:1272 pools row 0): M = B rows.  The LayerNorms are materialised
        // on the CLS rows and FFN1 runs on the plain (not gamma-scaled) weight.  The W2 residual adds `res`: post-LN the
        // LN1-normalised rows, pre-LN the raw sums; the output LayerNorm reads the new sums from `sum` and writes `res`.
        float *res = PRE_LN ? e->tmp_cls : e->x_cls, *sum = PRE_LN ? e->x_cls : e->tmp_cls;
        const int cb = (B + wpb - 1) / wpb;
        const PendingNorm p = pending_norm<PRE_LN>(e, c.layers - 1, false, e->stats_a);
        if (p.stats == e->stats_id)   // identity pending: pre-LN, or the embeddings of a single-layer encoder
            gather_cls_kernel<<<cb, wpb * 32, 0, s>>>(e->ctx, e->x, B, S, H, e->ctx_cls, e->x_cls);
        else
            gather_cls_ln_kernel<<<cb, wpb * 32, 0, s>>>(e->ctx, e->x, B, S, H, p.gamma, p.beta, c.ln_eps, e->ctx_cls, e->x_cls);
        AC_LAUNCH_CHECK();
        EpiF32<false, true> eo{.bias = last.bo, .residual = e->x_cls, .Y = e->tmp_cls, .M = B, .N = H, .ldy = H};
        if ((rc = launch_linear(e->m_ctx_cls, last.m_wo, B, H, H, eo, s))) return rc;
        layernorm_kernel<NORM><<<cb, wpb * 32, 0, s>>>(e->tmp_cls, last.ln_ffn_w, last.ln_ffn_b, c.ln_eps, B, H, PRE_LN ? nullptr : res,
                                                 e->xh_cls);
        AC_LAUNCH_CHECK();
        if ((rc = run_ffn1_rows<FFN_ACT>(e, e->m_xh_cls, e->ffn_cls, B, s))) return rc;
        EpiF32<false, true> e2{.bias = last.b2, .residual = res, .Y = sum, .M = B, .N = H, .ldy = H};
        if ((rc = launch_linear(e->m_ffn_cls, last.m_w2, B, H, I, e2, s))) return rc;
        layernorm_kernel<NORM><<<cb, wpb * 32, 0, s>>>(sum, last.ln_out_w, last.ln_out_b, c.ln_eps, B, H, res, nullptr);
        AC_LAUNCH_CHECK();
        if ((rc = launch_cls_normalize(res, B, 1, H, out_unit_cls, s))) return rc;
    } else {
        // full hidden state requested (cls_only = 0, or B > Bc): materialise the output LayerNorm for every row
        layernorm_kernel<NORM><<<row_blocks, wpb * 32, 0, s>>>(e->x, last.ln_out_w, last.ln_out_b, c.ln_eps, M, H, e->tmp, nullptr);
        AC_LAUNCH_CHECK();
        if ((rc = launch_cls_normalize(e->tmp, B, S, H, out_unit_cls, s))) return rc;
    }
    e->last_B = B;
    e->last_S = S;
    e->last_cls_only = cls_tail;
    return AC_OK;
}

// The block kind of a handle's architecture as forward_layers' template arguments: f(BlockKind<..>{}) with the handle's.
template <bool PRE_LN_, bool ROPE_, Act FFN_ACT_, Norm NORM_>
struct BlockKind {
    static constexpr bool PRE_LN = PRE_LN_, ROPE = ROPE_;
    static constexpr Act FFN_ACT = FFN_ACT_;
    static constexpr Norm NORM = NORM_;
};
template <class F>
static int with_block_kind(const ac_encoder *e, F &&f) {
    constexpr Norm LN = Norm::Layer;
    const ac_encoder_config &c = e->cfg;
    if (c.arch == AC_ARCH_MODERNBERT) return f(BlockKind<true, true, Act::GeGLU, LN>{});
    if (c.arch == AC_ARCH_EUROBERT) return f(BlockKind<true, true, Act::SwiGLU, Norm::Rms>{});
    if (c.arch == AC_ARCH_ROTARY) {
        if (c.ffn_act == AC_FFN_SWIGLU) return f(BlockKind<false, true, Act::SwiGLU, LN>{});
        if (c.ffn_act == AC_FFN_GELU_TANH) return f(BlockKind<false, true, Act::GeluTanh, LN>{});
        return f(BlockKind<false, true, Act::Gelu, LN>{});
    }
    if (c.ffn_act == AC_FFN_GELU_TANH) return f(BlockKind<false, false, Act::GeluTanh, LN>{});
    return f(BlockKind<false, false, Act::Gelu, LN>{});
}

// Shape checks every entry that runs attention shares, then the V^T view of a (B, S) call: rows (b, h, d), S_pad keys per
// row; box = 64 keys x 64 rows (one head of 64, or a head of 32 and its neighbour; rows past B*H read as zeros).  The view
// is cached on the handle, keyed on (B, S).
static int check_shape_map_vt(ac_encoder *e, const char *who, int B, int S) {
    AC_REQUIRE(B > 0 && S > 0, "%s: B=%d S=%d", who, B, S);
    if (e->cfg.arch == AC_ARCH_MODERNBERT) {
        // RoPE has no position table: any S up to the encoder's max_pos (<= AC_MODERNBERT_MAX_S) runs
        AC_REQUIRE(S <= e->cfg.max_pos, "%s: S=%d exceeds this ModernBERT encoder's max_pos=%d (max_position_embeddings)", who,
                   S, e->cfg.max_pos);
    } else if (e->cfg.arch == AC_ARCH_ROTARY) {
        AC_REQUIRE(S <= e->cfg.max_pos, "%s: S=%d exceeds this rotary encoder's max_pos=%d (min(max_position_embeddings, %d))",
                   who, S, e->cfg.max_pos, AC_MODERNBERT_MAX_S);
    } else if (e->cfg.arch == AC_ARCH_EUROBERT) {
        AC_REQUIRE(S <= e->cfg.max_pos, "%s: S=%d exceeds this EuroBERT encoder's max_pos=%d (min(max_position_embeddings, %d))",
                   who, S, e->cfg.max_pos, AC_MODERNBERT_MAX_S);
    } else if (e->cfg.arch == AC_ARCH_DEBERTA && e->cfg.rel_radius > AC_ENCODER_MAX_S) {
        // relative positions only (ac_encoder_create checked that pos_emb is zeros): rel_index bounds S, max_pos does not
        if (S > e->cfg.rel_radius) {
            set_error("%s: S=%d exceeds %d, the rel_radius of this DeBERTa encoder's relative position index", who, S,
                      e->cfg.rel_radius);
            return AC_E_UNSUPPORTED;
        }
    } else if (S > AC_ENCODER_MAX_S) {
        // RoBERTa positions run from pad_idx + 1: a table with more rows than AC_ENCODER_MAX_S of them (XLM-R's 8194) takes
        // the sequences it has positions for, up to AC_MODERNBERT_MAX_S
        const ac_encoder_config &c = e->cfg;
        if (c.arch != AC_ARCH_ROBERTA || c.max_pos <= AC_ENCODER_MAX_S + c.pad_idx + 1) {
            set_error("%s: S=%d > 512 is not supported (the reference truncates at max_length = 512)", who, S);
            return AC_E_UNSUPPORTED;
        }
        const int s_max = std::min(AC_MODERNBERT_MAX_S, c.max_pos - c.pad_idx - 1);
        if (S > s_max) {
            set_error("%s: S=%d exceeds %d, the longest sequence this RoBERTa encoder has positions for "
                      "(max_position_embeddings=%d, positions from pad_idx + 1 = %d, at most %d)",
                      who, S, s_max, c.max_pos, c.pad_idx + 1, AC_MODERNBERT_MAX_S);
            return AC_E_UNSUPPORTED;
        }
    }
    AC_REQUIRE(static_cast<int64_t>(B) * S <= e->cfg.max_tokens, "%s: B*S=%lld exceeds max_tokens=%d", who,
               static_cast<long long>(B) * S, e->cfg.max_tokens);
    AC_REQUIRE(S <= e->cfg.max_pos || e->cfg.rel_radius > AC_ENCODER_MAX_S, "%s: S exceeds max_position_embeddings", who);
    const int H = e->cfg.hidden;
    const int S_pad = (S + 7) / 8 * 8;
    AC_REQUIRE(static_cast<size_t>(B) * H * S_pad <= e->vt_elems,
               "%s: B=%d sequences of S=%d exceed the transposed-V workspace; split the batch", who, B, S);
    if (e->vt_B != B || e->vt_S != S) {
        int rc = make_tmap_2d(&e->m_vt_att, e->vT, 2, static_cast<uint64_t>(B) * H, S_pad, static_cast<uint64_t>(S_pad) * 2, 64, 64);
        if (rc) return rc;
        e->vt_B = B; e->vt_S = S;
    }
    return AC_OK;
}

extern "C" int ac_encoder_forward_cls(ac_encoder *e, const int32_t *ids, const int32_t *mask, const int32_t *type_ids,
                                      int B, int S, float *out_unit_cls, ac_stream_t stream) {
    AC_REQUIRE(e && ids && out_unit_cls, "ac_encoder_forward_cls: null argument");
    int rc = check_shape_map_vt(e, "ac_encoder_forward_cls", B, S);
    if (rc) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return with_block_kind(e, [&](auto k) {
        using K = decltype(k);
        return forward_layers<K::PRE_LN, K::ROPE, K::FFN_ACT, K::NORM>(e, ids, mask, type_ids, B, S, out_unit_cls, s);
    });
}

// parity entry: one projection role of layer `layer` on caller-supplied inputs, through the handle's own packed operands,
// buffers and the role functions forward_layers runs (include/adaptive_b200.h)
extern "C" int ac_encoder_projection(ac_encoder *e, int layer, int role, int B, int S, const void *a, const float *y,
                                     const float *stats, void *out0, void *out1, float *stats_out, ac_stream_t stream) {
    AC_REQUIRE(e && a && out0, "ac_encoder_projection: null argument");
    const ac_encoder_config &c = e->cfg;
    AC_REQUIRE(role >= AC_PROJ_EMB && role <= AC_PROJ_FFN1_ROWS, "ac_encoder_projection: unknown role=%d", role);
    AC_REQUIRE(layer >= 0 && layer < c.layers, "ac_encoder_projection: layer=%d outside 0..%d", layer, c.layers - 1);
    AC_REQUIRE(role != AC_PROJ_EMB || e->emb_proj_w, "ac_encoder_projection: AC_PROJ_EMB needs an encoder with an embedding "
                                                     "projection (emb_proj_w)");
    AC_REQUIRE(role != AC_PROJ_FFN1_ROWS || c.cls_only, "ac_encoder_projection: AC_PROJ_FFN1_ROWS needs a cls_only encoder");
    AC_REQUIRE(B > 0 && S > 0 && static_cast<int64_t>(B) * S <= c.max_tokens,
               "ac_encoder_projection: B=%d S=%d: B*S must be in 1..max_tokens=%d", B, S, c.max_tokens);
    const bool resid = role == AC_PROJ_WO || role == AC_PROJ_W2;
    AC_REQUIRE((role == AC_PROJ_EMB || role == AC_PROJ_FFN1_ROWS || stats) && (!resid || (y && stats_out)) &&
                   (role == AC_PROJ_FFN1 || role == AC_PROJ_FFN1_ROWS || out1),
               "ac_encoder_projection: role=%d lacks one of stats, y, out1, stats_out", role);
    int rc;
    if (role == AC_PROJ_QKV && (rc = check_shape_map_vt(e, "ac_encoder_projection", B, S))) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t M = static_cast<size_t>(B) * S, H = c.hidden, I = c.intermediate, h2 = sizeof(__half);
    const auto copy = [&](void *dst, const void *src, size_t bytes) {
        return check_cuda(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s), "ac_encoder_projection copy");
    };
    const float2 *st_in = reinterpret_cast<const float2 *>(stats);
    return with_block_kind(e, [&](auto k) -> int {
        using K = decltype(k);
        int rc;
        switch (role) {
        case AC_PROJ_EMB:
            if ((rc = copy(e->ctx, a, M * c.embedding_size * h2)) || (rc = run_emb_proj(e, static_cast<int>(M), s)) ||
                (rc = copy(out0, e->x, M * H * sizeof(float))))
                return rc;
            return copy(out1, e->xh, M * H * h2);
        case AC_PROJ_QKV:
            if ((rc = copy(e->xh, a, M * H * h2)) || (rc = copy(e->stats_a, stats, M * sizeof(float2))) ||
                (rc = run_qkv<K::ROPE>(e, layer, B, S, e->stats_a, s)) || (rc = copy(out0, e->qk, M * 2 * H * h2)))
                return rc;
            return copy(out1, e->vT, B * H * ((S + 7) / 8 * 8) * h2);
        case AC_PROJ_FFN1:
            if ((rc = copy(e->xh, a, M * H * h2)) || (rc = copy(e->stats_b, stats, M * sizeof(float2))) ||
                (rc = run_ffn1<K::FFN_ACT>(e, layer, static_cast<int>(M), e->stats_b, s)))
                return rc;
            return copy(out0, e->ffn, M * I * h2);
        case AC_PROJ_FFN1_ROWS:
            AC_REQUIRE(layer == c.layers - 1, "ac_encoder_projection: AC_PROJ_FFN1_ROWS is the last layer's (layer=%d)", layer);
            if ((rc = copy(e->xh, a, M * H * h2)) || (rc = run_ffn1_rows<K::FFN_ACT>(e, e->m_xh, e->ffn, static_cast<int>(M), s)))
                return rc;
            return copy(out0, e->ffn, M * I * h2);
        default: {   // AC_PROJ_WO, AC_PROJ_W2: the residual sums y and their statistics in, the new sums and theirs out
            const bool ffn = role == AC_PROJ_W2;
            float2 *st = ffn ? e->stats_b : e->stats_a;
            if ((rc = copy(ffn ? e->ffn : e->ctx, a, M * (ffn ? I : H) * h2)) || (rc = copy(e->x, y, M * H * sizeof(float))) ||
                (rc = copy(st, st_in, M * sizeof(float2))) ||
                (rc = run_resid<K::PRE_LN, K::NORM>(e, layer, ffn, static_cast<int>(M), st, ffn ? e->stats_a : e->stats_b, s)) ||
                (rc = copy(out0, e->x, M * H * sizeof(float))) || (rc = copy(out1, e->xh, M * H * h2)))
                return rc;
            return copy(stats_out, ffn ? e->stats_a : e->stats_b, M * sizeof(float2));
        }
        }
    });
}

// parity entry: the attention stage alone, through the handle's own buffers, V^T view and launch_attention
extern "C" int ac_encoder_attention(ac_encoder *e, const void *qk, const void *vT, const int32_t *mask, int B, int S, int window,
                                    int cls_rows, void *ctx_out, ac_stream_t stream) {
    AC_REQUIRE(e && qk && vT && ctx_out, "ac_encoder_attention: null argument");
    AC_REQUIRE(window >= 0 && (window == 0 || e->cfg.arch == AC_ARCH_MODERNBERT),
               "ac_encoder_attention: window=%d needs an AC_ARCH_MODERNBERT encoder (0 = full attention)", window);
    int rc = check_shape_map_vt(e, "ac_encoder_attention", B, S);
    if (rc) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t H = e->cfg.hidden, M = static_cast<size_t>(B) * S, S_pad = (S + 7) / 8 * 8;
    AC_CUDA(cudaMemcpyAsync(e->qk, qk, M * 2 * H * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    AC_CUDA(cudaMemcpyAsync(e->vT, vT, B * H * S_pad * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    if ((rc = launch_attention(e, mask, B, S, window, cls_rows != 0, 0, s))) return rc;
    AC_CUDA(cudaMemcpyAsync(ctx_out, e->ctx, M * H * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    return AC_OK;
}

extern "C" int ac_encoder_last_hidden(ac_encoder *e, float *out, int64_t n_floats, ac_stream_t stream) {
    AC_REQUIRE(e && out, "ac_encoder_last_hidden: null argument");
    AC_REQUIRE(!e->last_cls_only, "ac_encoder_last_hidden: the previous forward computed only the CLS rows of the last layer "
                                  "(create the encoder with cls_only = 0 to keep the full hidden state)");
    const int64_t have = static_cast<int64_t>(e->last_B) * e->last_S * e->cfg.hidden;
    AC_REQUIRE(n_floats <= have, "ac_encoder_last_hidden: asked %lld floats, have %lld", (long long)n_floats, (long long)have);
    AC_CUDA(cudaMemcpyAsync(out, e->tmp, n_floats * sizeof(float), cudaMemcpyDeviceToDevice,
                            static_cast<cudaStream_t>(stream)));
    return AC_OK;
}

// generic tensor-core linear exposed for parity tests / roofline measurement (the encoder's GEMM with a plain epilogue).
//   precision AC_PREC_TF32: X, W fp32 (used as stored, tf32 truncation by the MMA unless pre-rounded), Y fp32
//   precision AC_PREC_F16 : X, W fp16, Y fp32 (out_half = 0) or fp16 (out_half = 1)
template <int KIND>
static int linear_tc(const CUtensorMap &ta, const CUtensorMap &tb, const float *bias, const float *residual, void *Y, int M,
                     int N, int K, int epi, int round_out, int out_half, cudaStream_t s) {
    const auto run = [&](const auto &e) {
        return launch_gemm_tc<std::decay_t<decltype(e)>, false, KIND>(ta, tb, M, N, K, e, s);
    };
    if constexpr (KIND == GEMM_KIND_F16) {
        if (out_half) {
            __half *Yh = static_cast<__half *>(Y);
            if (epi == 0) return run(EpiF16<Act::None, false>{.bias = bias, .Y = Yh, .M = M, .N = N, .ldy = N});
            if (epi == 3) return run(EpiF16<Act::GeluTanh, false>{.bias = bias, .Y = Yh, .M = M, .N = N, .ldy = N});
            if (epi == 4) return run(EpiF16<Act::SwiGLU, false>{.bias = bias, .Y = Yh, .M = M, .N = N, .ldy = N / 2});
            return run(EpiF16<Act::Gelu, false>{.bias = bias, .Y = Yh, .M = M, .N = N, .ldy = N});
        }
    }
    float *Yf = static_cast<float *>(Y);
    if (epi == 0) return run(EpiF32<false, false>{.bias = bias, .Y = Yf, .M = M, .N = N, .ldy = N, .round_out = round_out});
    if (epi == 1) return run(EpiF32<true, false>{.bias = bias, .Y = Yf, .M = M, .N = N, .ldy = N, .round_out = round_out});
    return run(EpiF32<false, true>{.bias = bias, .residual = residual, .Y = Yf, .M = M, .N = N, .ldy = N,
                                   .round_out = round_out});
}

extern "C" int ac_linear_tc(const void *X, const void *W, const float *bias, const float *residual, void *Y, int M, int N,
                            int K, int epi, int round_out, int precision, int out_half, ac_stream_t stream) {
    AC_REQUIRE(X && W && Y && bias && M > 0 && N > 0 && K > 0, "ac_linear_tc: bad arguments (bias is required)");
    AC_REQUIRE(epi >= 0 && epi <= 4 && (epi != 2 || residual), "ac_linear_tc: bad epilogue");
    AC_REQUIRE(precision == AC_PREC_TF32 || precision == AC_PREC_F16, "ac_linear_tc: bad precision");
    AC_REQUIRE(!(out_half && epi == 2), "ac_linear_tc: the residual epilogue writes fp32");
    AC_REQUIRE(epi != 3 || (out_half && precision == AC_PREC_F16), "ac_linear_tc: the tanh-GELU epilogue writes fp16");
    AC_REQUIRE(epi != 4 || (out_half && precision == AC_PREC_F16 && N % 64 == 0),
               "ac_linear_tc: the SwiGLU epilogue writes fp16 and takes N %% 64 == 0 (interleaved weight rows)");
    const int es = precision == AC_PREC_F16 ? 2 : 4;
    AC_REQUIRE((K * es) % 16 == 0 && N % 8 == 0, "ac_linear_tc: rows must be 16-byte multiples and N %% 8 == 0");
    int rc = ac_device_check();
    if (rc) return rc;
    CUtensorMap ta, tb;
    const uint32_t bk = 128 / es;
    if ((rc = make_tmap_2d(&ta, X, es, M, K, static_cast<uint64_t>(K) * es, GEMM_BLOCK_M, bk))) return rc;
    if ((rc = make_tmap_2d(&tb, W, es, N, K, static_cast<uint64_t>(K) * es, GEMM_BLOCK_N, bk))) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (precision == AC_PREC_TF32) {
        AC_REQUIRE(!out_half, "ac_linear_tc: tf32 path writes fp32");
        return linear_tc<GEMM_KIND_TF32>(ta, tb, bias, residual, Y, M, N, K, epi, round_out, 0, s);
    }
    return linear_tc<GEMM_KIND_F16>(ta, tb, bias, residual, Y, M, N, K, epi, 0, out_half, s);
}
