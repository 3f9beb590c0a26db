// Internal kernel-launch interface of libwisb200.so (host side). One .cu per kernel family.
#pragma once
#include "common.cuh"

namespace wisb {

// ------------------------------------------------------------------ wgmma GEMM  (gemm_tc.cu)
// D[M,N] = A[M,K] . W[N,K]^T, fp16 operands (both K-major), fp32 accumulation in registers, fused epilogues.
enum EpiMode : int {
  EPI_F16 = 0,        // out16[row, col] = acc + bias
  EPI_F16_GELU = 1,   // out16 = gelu(acc + bias)
  EPI_RESID_F32 = 2,  // out32[row, col] += acc + bias           (residual stream, in place)
  EPI_CONV2 = 3,      // out32 = gelu(acc + bias) + pos[row % 1536, col]   (conv2 of the stem; rows >= 1500 get 0)
  EPI_CROSSKV = 4,    // out16 scattered to [layer][k|v][b][head][1536][64]
  EPI_F32 = 5,        // out32 = acc (+ bias)
  EPI_QKV_VT = 6,     // cols < 2d: out16 = acc + bias; cols >= 2d (V): aux16[b][head][e][t] = acc + bias (transposed)
  EPI_DEC_QKV = 7,    // batched decoder pass: cols < d: out32 (q) = acc + bias; K / V columns go to the self-attention
                      // cache rows [(row_slot[row] * t_cap + row_pos[row]) * d + e] of aux (K) / aux2 (V) as fp16
};

struct GemmEpi {
  int mode = EPI_F16;
  const float* bias = nullptr;  // [N] or null
  void* out = nullptr;
  long long ldo = 0;   // leading dimension of out, elements
  int m_valid = 0;     // rows >= m_valid are not written
  int n_valid = 0;     // cols >= n_valid are not written (multiple of 32)
  const float* pos = nullptr;  // EPI_CONV2: [1500, N] float32
  void* aux = nullptr;         // EPI_QKV_VT: Vt buffer; EPI_DEC_QKV: K cache of the layer
  void* aux2 = nullptr;        // EPI_DEC_QKV: V cache of the layer
  int d_model = 0, n_heads = 0, batch = 0;  // EPI_CROSSKV / EPI_QKV_VT
  int batch_off = 0;           // EPI_CROSSKV: window b of this call is utterance batch_off + b of the `batch`-wide K/V buffer
  int kv_swizzle = 0;          // EPI_CROSSKV: 16-byte chunks of a key row XOR-swizzled by the key index (warp-MMA decoder pass)
  const int* row_slot = nullptr;  // EPI_DEC_QKV: cache slot / position of every row (device arrays)
  const int* row_pos = nullptr;
  int t_cap = 0;               // EPI_DEC_QKV: positions per cache slot
  long long split_stride = 0;  // split-K (EPI_F32 only): partial of split s goes to out + s * split_stride elements
  const int* m_dyn = nullptr;  // optional device-side row count: M tiles at or beyond it are skipped
};

struct GemmPlan {
  CUtensorMap map_a, map_b;
  int M = 0, N = 0, K = 0, BN = 128, grid = 0, a_wrap = 0, mcast = 0, k_splits = 1, pdl = 0;
  GemmEpi epi;
};

// A: M rows of K fp16, row r starts at a + r * lda (lda in elements; may be < K for the overlapping-row view conv2 uses)
// a_wrap > 0 (conv2): A is stored as rows of `a_wrap` (= lda) elements and logical row r continues into row r + 1.
void gemm_plan(GemmPlan& p, const __half* a, long long lda, const __half* w, int M, int N, int K, const GemmEpi& epi,
               int num_sms, int force_bn = 0, int a_wrap = 0, int k_splits = 1);
// (force_bn < 0: same |force_bn| tile but without the 2-CTA multicast clusters -- diagnostics)
void gemm_run(const GemmPlan& p, cudaStream_t stream);
// slow SIMT cross-check used only by the diagnostics entry point / tests
void gemm_ref_run(const __half* a, long long lda, const __half* w, float* c, int M, int N, int K, cudaStream_t stream);

// 2-D fp16 tensor map: inner dimension `cols` (contiguous), `rows` rows of stride `ld` elements, 128B swizzle
void make_tmap_f16_2d(CUtensorMap* map, const void* ptr, long long cols, long long rows, long long ld, int box_cols,
                      int box_rows);

// ------------------------------------------------------------------ log-mel front end (logmel.cu)
// pcm: B utterances, f32 or s16, utterance b starts at pcm + offsets[b] (elements) and has n_samples[b] samples
// (unpadded; padding / trimming to 480000 is fused).  mel: [B, 80, 3000] f32 on device.
size_t logmel_table_floats();
void logmel_init_tables(float* tables_dev, cudaStream_t stream);
void logmel_run(const void* pcm, int pcm_is_s16, const long long* offsets_dev, const int* n_samples_dev, int B,
                const float* tables_dev, float* mel, unsigned* max_ws /* [B] */, cudaStream_t stream);

// ------------------------------------------------------------------ encoder pieces (encoder.cu)
// conv1 (80 -> d, k=3, pad 1) + GELU, writes h1 [B, 3072, d] fp16 with the row layout conv2's strided view needs
void conv1_gelu_run(const float* mel, const __half* w /*[d,240]*/, const float* bias, __half* h1, int B, int d,
                    cudaStream_t stream);
// LayerNorm over rows of fp32 x [rows, d] -> fp16 y [rows, d]
void layernorm_f32_to_f16_run(const float* x, const float* g, const float* b, __half* y, int rows, int d,
                              cudaStream_t stream, bool pdl = false);
// non-causal self-attention over the 1500 valid positions of each window; qkv [B*1536, 3d] fp16 -> ctx [B*1536, d] fp16
struct AttnPlan {
  CUtensorMap map_q, map_k, map_v;
  int B = 0, d = 0, H = 0;
  bool v_mn_major = true;
  bool pdl = false;  // programmatic dependent launch (the kernel's prologue overlaps its predecessor's tail)
  __half* ctx = nullptr;
};
void enc_attn_plan(AttnPlan& p, const __half* qkv, const __half* vt, __half* ctx, int B, int d, int H, bool v_mn_major);
void enc_attn_run(const AttnPlan& p, cudaStream_t stream);
// SIMT cross-check of the same attention (diagnostics only)
void enc_attn_ref_run(const __half* qkv, __half* ctx, int B, int d, int H, cudaStream_t stream);

}  // namespace wisb
