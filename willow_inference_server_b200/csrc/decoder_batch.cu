// Batched decoder pass: ONE pass over the decoder weights serves every row (utterance x beam) of a batch of utterances.
//
// Reference semantics: the decoder step of ctranslate2.models.Whisper.generate for a batch of feature windows
// (main.py:676-693 of the reference server feeds several windows per call; SURVEY.md section 8a row A10, section 7 step 5:
// "decoder with M = B x beam rows").  Architecture per [HF] modeling_whisper.py:417-508.
//
// Up to 8 rows the persistent passes (decoder_mega.cu) are the latency path.  Beyond that the pass is a chain of
//   * wgmma GEMMs (gemm_tc.cu): rows are the M dimension (padded to 128-row tiles), the weight matrix streams through
//     the TMA ring exactly once per pass whatever the number of rows; narrow tiles (BN = 64) and split-K keep >= ~100 CTAs
//     streaming even when the weight matrix has only d_model output columns;
//   * the small kernels below: embedding + LayerNorm, split-K reduction + bias + residual + LayerNorm (one kernel),
//     self-attention over the beam-indirected cache, cross-attention that reads each utterance's K/V once for all beams.
// The whole chain (+ the search kernels) is captured in one CUDA graph per batch shape by the engine.
// Activations feeding a GEMM are fp16 (tensor-core operands), the residual stream and all reductions are fp32.
#include <cooperative_groups.h>

#include "decoder.cuh"
#include "ptx.cuh"

namespace cg = cooperative_groups;

namespace wisb {

namespace {

constexpr int BD_LN_WARPS = 4;   // rows per CTA (one warp per row: no block-level synchronisation at all)
constexpr int BD_LN_MAX = 12;    // float4 per lane: d_model <= 1536

// LayerNorm of the warp's row held in registers (v[i] = float4 number lane + 32 i of the row) -> fp16;
// two-pass statistics in fp32 (mean, then the centred sum of squares), as torch.nn.functional.layer_norm does
__device__ __forceinline__ void row_layernorm_store(const float4 (&v)[BD_LN_MAX], int iters, int d, const float* __restrict__ g,
                                                    const float* __restrict__ b, __half* __restrict__ out, int lane) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < BD_LN_MAX; ++i)
    if (i < iters) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) / d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < BD_LN_MAX; ++i)
    if (i < iters) {
      const float a0 = v[i].x - mean, a1 = v[i].y - mean, a2 = v[i].z - mean, a3 = v[i].w - mean;
      q += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
    }
  const float rstd = rsqrtf(warp_sum(q) / d + 1e-5f);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const float4* b4 = reinterpret_cast<const float4*>(b);
  uint2* o2 = reinterpret_cast<uint2*>(out);
#pragma unroll
  for (int i = 0; i < BD_LN_MAX; ++i)
    if (i < iters) {
      const float4 gg = __ldg(g4 + i * 32 + lane), bb = __ldg(b4 + i * 32 + lane);
      __half2 h0 = __floats2half2_rn((v[i].x - mean) * rstd * gg.x + bb.x, (v[i].y - mean) * rstd * gg.y + bb.y);
      __half2 h1 = __floats2half2_rn((v[i].z - mean) * rstd * gg.z + bb.z, (v[i].w - mean) * rstd * gg.w + bb.w);
      uint2 u;
      u.x = *reinterpret_cast<uint32_t*>(&h0);
      u.y = *reinterpret_cast<uint32_t*>(&h1);
      o2[i * 32 + lane] = u;
    }
}

// x[r] = tok_emb[token[r]] + pos_emb[row_pos[r]];  xn[r] = LN(x[r])   (first LayerNorm of decoder layer 0)
__global__ void __launch_bounds__(BD_LN_WARPS * 32)
bd_embed_ln_kernel(const int* __restrict__ tokens, const int* __restrict__ row_pos, const __half* __restrict__ tok_emb,
                   const float* __restrict__ pos_emb, const float* __restrict__ g, const float* __restrict__ b,
                   float* __restrict__ x, __half* __restrict__ xn, int d, int rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * BD_LN_WARPS + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int iters = d / 128;
  const uint2* e2 = reinterpret_cast<const uint2*>(tok_emb + static_cast<long long>(tokens[r]) * d);
  const float4* p4 = reinterpret_cast<const float4*>(pos_emb + static_cast<long long>(row_pos[r]) * d);
  float4* x4 = reinterpret_cast<float4*>(x + static_cast<long long>(r) * d);
  float4 v[BD_LN_MAX];
#pragma unroll
  for (int i = 0; i < BD_LN_MAX; ++i)
    if (i < iters) {
      const uint2 eu = __ldg(e2 + i * 32 + lane);
      const float4 pp = __ldg(p4 + i * 32 + lane);
      const float2 e01 = __half22float2(*reinterpret_cast<const __half2*>(&eu.x));
      const float2 e23 = __half22float2(*reinterpret_cast<const __half2*>(&eu.y));
      v[i] = make_float4(e01.x + pp.x, e01.y + pp.y, e23.x + pp.z, e23.y + pp.w);
      x4[i * 32 + lane] = v[i];
    }
  row_layernorm_store(v, iters, d, g, b, xn + static_cast<long long>(r) * d, lane);
}

// x[r] += bias + sum_s partial[s][r]  (split-K slabs of the preceding GEMM, fixed summation order);  xn[r] = LN(x[r])
template <int NS>
__global__ void __launch_bounds__(BD_LN_WARPS * 32)
bd_resid_ln_kernel(float* __restrict__ x, const float* __restrict__ partial, long long split_stride,
                   const float* __restrict__ bias, const float* __restrict__ g, const float* __restrict__ b,
                   __half* __restrict__ xn, int d, int rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * BD_LN_WARPS + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int iters = d / 128;
  float4* x4 = reinterpret_cast<float4*>(x + static_cast<long long>(r) * d);
  const float4* b4 = reinterpret_cast<const float4*>(bias);
  float4 v[BD_LN_MAX];
#pragma unroll
  for (int i = 0; i < BD_LN_MAX; ++i)
    if (i < iters) {
      // every load of this float4 is issued before the first add: one round trip per element whatever the split count
      const float4 xv = x4[i * 32 + lane];
      const float4 bv = __ldg(b4 + i * 32 + lane);
      float4 pv[NS];
#pragma unroll
      for (int s = 0; s < NS; ++s)
        pv[s] = __ldcg(reinterpret_cast<const float4*>(partial + s * split_stride + static_cast<long long>(r) * d) + i * 32 + lane);
      float4 acc = bv;
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        acc.x += pv[s].x; acc.y += pv[s].y; acc.z += pv[s].z; acc.w += pv[s].w;
      }
      v[i] = make_float4(xv.x + acc.x, xv.y + acc.y, xv.z + acc.z, xv.w + acc.w);
      x4[i * 32 + lane] = v[i];
    }
  row_layernorm_store(v, iters, d, g, b, xn + static_cast<long long>(r) * d, lane);
}

// =====================================================================================================================
// self-attention over the cache: one warp per (row, head).  Position t < pos of row r lives in cache slot indir[r][t]
// (beam reordering by indirection, search.cu), position pos in the row's own slot (written by this pass's QKV GEMM).
// Prefill rows (prompt positions of one utterance, all in the utterance's first slot) attend their own slot only.
// =====================================================================================================================
constexpr int BD_SA_TMAX = 448;

__global__ void __launch_bounds__(128)
bd_self_attn_kernel(const float* __restrict__ q, const __half* __restrict__ kcache, const __half* __restrict__ vcache,
                    const int* __restrict__ row_pos, const int* __restrict__ row_slot, const int* __restrict__ indir0,
                    const int* __restrict__ indir1, const int* __restrict__ flip, const int* __restrict__ done,
                    __half* __restrict__ ctx, int d, int H, int t_cap, int t_ind, int rows_per_utt, int prefill) {
  __shared__ float s_p[4][BD_SA_TMAX];
  __shared__ int s_slot[4][BD_SA_TMAX];
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x * 4 + warp;
  const int r = blockIdx.y;
  if (h >= H) return;
  if (done != nullptr && done[r / rows_per_utt]) return;  // finished utterance: its rows are dead weight
  const int pos = row_pos[r];
  const int own = row_slot[r];
  const int* indir = (*flip ? indir1 : indir0) + static_cast<long long>(r) * t_ind;
  const float* qr = q + static_cast<long long>(r) * d + h * HEAD_DIM;
  float qv[HEAD_DIM];
#pragma unroll
  for (int i = 0; i < HEAD_DIM / 4; ++i) {
    const float4 v = *reinterpret_cast<const float4*>(qr + 4 * i);
    qv[4 * i] = v.x; qv[4 * i + 1] = v.y; qv[4 * i + 2] = v.z; qv[4 * i + 3] = v.w;
  }
  float mx = -INFINITY;
  for (int t = lane; t <= pos; t += 32) {
    const int slot = (prefill || t == pos) ? own : indir[t];
    s_slot[warp][t] = slot;
    const uint4* kr = reinterpret_cast<const uint4*>(kcache + (static_cast<long long>(slot) * t_cap + t) * d + h * HEAD_DIM);
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint4 u = kr[i];
      const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h2[j]);
        s0 = fmaf(qv[8 * i + 2 * j], f.x, s0);
        s1 = fmaf(qv[8 * i + 2 * j + 1], f.y, s1);
      }
    }
    const float s = (s0 + s1) * 0.125f;
    s_p[warp][t] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int t = lane; t <= pos; t += 32) {
    const float p = __expf(s_p[warp][t] - mx);
    s_p[warp][t] = p;
    sum += p;
  }
  sum = warp_sum(sum);
  __syncwarp();
  float o0 = 0.f, o1 = 0.f;
  for (int t = 0; t <= pos; ++t) {
    const float p = s_p[warp][t];
    const __half2 v = *reinterpret_cast<const __half2*>(vcache + (static_cast<long long>(s_slot[warp][t]) * t_cap + t) * d +
                                                        h * HEAD_DIM + 2 * lane);
    const float2 f = __half22float2(v);
    o0 = fmaf(p, f.x, o0);
    o1 = fmaf(p, f.y, o1);
  }
  const float inv = 1.0f / sum;
  *reinterpret_cast<__half2*>(ctx + static_cast<long long>(r) * d + h * HEAD_DIM + 2 * lane) = __floats2half2_rn(o0 * inv, o1 * inv);
}

// =====================================================================================================================
// cross-attention: one cluster of 8 CTAs per (head, utterance); CTA c owns keys [192 c, 192 c + 192) of the 1536-row
// padded window (keys >= 1500 are skipped).  Inside a CTA, groups of 8 lanes walk keys with an online softmax for all
// rows of the utterance at once -- the utterance's K/V (251.7 MB over the layers at large-v2) are read ONCE per pass for
// every beam -- partials are merged through shared memory, and the 8 CTAs merge through distributed shared memory.
// Finished utterances are skipped: their K/V are not read at all.
// =====================================================================================================================
constexpr int BD_CA_CLUSTER = 8;
constexpr int BD_CA_KEYS = T_ENC_PAD / BD_CA_CLUSTER;  // 192
constexpr int BD_CA_THREADS = 128;
constexpr int BD_CA_GROUPS = BD_CA_THREADS / 8;        // 16 groups of 8 lanes; 12 keys each

template <int NB>
__global__ void __cluster_dims__(1, 1, BD_CA_CLUSTER) __launch_bounds__(BD_CA_THREADS)
bd_cross_attn_kernel(const float* __restrict__ q, const __half* __restrict__ kmat, const __half* __restrict__ vmat,
                     const int* __restrict__ done, __half* __restrict__ ctx, int rows_per_utt, int d, int H) {
  // dynamic smem: [K tile 192 x 64 fp16 | V tile 192 x 64 fp16 | per-group partial accumulators]
  extern __shared__ __align__(128) uint8_t ca_smem[];
  __half* sK = reinterpret_cast<__half*>(ca_smem);
  __half* sV = sK + BD_CA_KEYS * HEAD_DIM;
  float (*s_acc)[NB][HEAD_DIM] = reinterpret_cast<float (*)[NB][HEAD_DIM]>(ca_smem + 2 * BD_CA_KEYS * HEAD_DIM * 2);
  __shared__ float s_m[BD_CA_GROUPS][NB], s_l[BD_CA_GROUPS][NB];
  __shared__ float c_acc[NB][HEAD_DIM];  // this CTA's merged partial (read by the cluster leader through DSMEM)
  __shared__ float c_m[NB], c_l[NB];
  __shared__ uint64_t s_bar;
  cg::cluster_group cluster = cg::this_cluster();
  const int h = blockIdx.x, u = blockIdx.y, cta = blockIdx.z;
  const int tid = threadIdx.x;
  pdl_launch_dependents();
  const int grp = tid >> 3, gl = tid & 7;  // lane gl of group grp owns dims [8 gl, 8 gl + 8)
  const long long head_off = (static_cast<long long>(u) * H + h) * T_ENC_PAD * HEAD_DIM;
  const int t_begin = cta * BD_CA_KEYS;
  const uint32_t bar = smem_u32(&s_bar);
  if (tid == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  pdl_wait();  // q (and the `done` flags) come from the previous kernels of the chain
  if (done != nullptr && done[u]) return;  // uniform over the cluster: no CTA of it reaches cluster.sync()
  // one elected thread streams this CTA's 192 keys and values (2 x 24 KB, contiguous) into shared memory with TMA
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, 2u * BD_CA_KEYS * HEAD_DIM * 2u);
    bulk_load_1d(smem_u32(sK), kmat + head_off + static_cast<long long>(t_begin) * HEAD_DIM, BD_CA_KEYS * HEAD_DIM * 2, bar);
    bulk_load_1d(smem_u32(sV), vmat + head_off + static_cast<long long>(t_begin) * HEAD_DIM, BD_CA_KEYS * HEAD_DIM * 2, bar);
  }
  float qv[NB][8];
#pragma unroll
  for (int k = 0; k < NB; ++k) {
    if (k < rows_per_utt) {
      const float* qr = q + static_cast<long long>(u * rows_per_utt + k) * d + h * HEAD_DIM + gl * 8;
      const float4 a0 = *reinterpret_cast<const float4*>(qr), a1 = *reinterpret_cast<const float4*>(qr + 4);
      qv[k][0] = a0.x * 0.125f; qv[k][1] = a0.y * 0.125f; qv[k][2] = a0.z * 0.125f; qv[k][3] = a0.w * 0.125f;
      qv[k][4] = a1.x * 0.125f; qv[k][5] = a1.y * 0.125f; qv[k][6] = a1.z * 0.125f; qv[k][7] = a1.w * 0.125f;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) qv[k][i] = 0.f;
    }
  }
  __syncthreads();  // barrier init visible
  mbar_wait(bar, 0);
  float m[NB], l[NB], acc[NB][8];
#pragma unroll
  for (int k = 0; k < NB; ++k) {
    m[k] = -INFINITY;
    l[k] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[k][i] = 0.f;
  }
  const unsigned gmask = 0xFFu << (tid & 24);  // the 8 lanes of this group (shuffles stay inside it)
#pragma unroll 1
  for (int tl = grp; tl < BD_CA_KEYS; tl += BD_CA_GROUPS) {
    if (t_begin + tl >= T_ENC) break;  // uniform inside the 8-lane group
    const uint4 ku = *reinterpret_cast<const uint4*>(sK + tl * HEAD_DIM + gl * 8);
    const uint4 vu = *reinterpret_cast<const uint4*>(sV + tl * HEAD_DIM + gl * 8);
    float kf[8], vf[8];
    {
      const __half2* k2 = reinterpret_cast<const __half2*>(&ku);
      const __half2* v2 = reinterpret_cast<const __half2*>(&vu);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 a = __half22float2(k2[i]), b = __half22float2(v2[i]);
        kf[2 * i] = a.x; kf[2 * i + 1] = a.y;
        vf[2 * i] = b.x; vf[2 * i + 1] = b.y;
      }
    }
#pragma unroll
    for (int k = 0; k < NB; ++k) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s = fmaf(qv[k][i], kf[i], s);
      s += __shfl_xor_sync(gmask, s, 1);
      s += __shfl_xor_sync(gmask, s, 2);
      s += __shfl_xor_sync(gmask, s, 4);
      const float mn = fmaxf(m[k], s);
      const float al = __expf(m[k] - mn), p = __expf(s - mn);
      l[k] = l[k] * al + p;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[k][i] = fmaf(acc[k][i], al, p * vf[i]);
      m[k] = mn;
    }
  }
#pragma unroll
  for (int k = 0; k < NB; ++k) {
#pragma unroll
    for (int i = 0; i < 8; ++i) s_acc[grp][k][gl * 8 + i] = acc[k][i];
    if (gl == 0) {
      s_m[grp][k] = m[k];
      s_l[grp][k] = l[k];
    }
  }
  __syncthreads();
  // merge the 16 groups: thread (k, e) pairs
  for (int idx = tid; idx < NB * HEAD_DIM; idx += BD_CA_THREADS) {
    const int k = idx / HEAD_DIM, e = idx % HEAD_DIM;
    float mm = -INFINITY;
    for (int g = 0; g < BD_CA_GROUPS; ++g) mm = fmaxf(mm, s_m[g][k]);
    float a = 0.f, ll = 0.f;
    for (int g = 0; g < BD_CA_GROUPS; ++g) {
      const float w = (s_m[g][k] == -INFINITY) ? 0.f : __expf(s_m[g][k] - mm);
      a = fmaf(w, s_acc[g][k][e], a);
      ll = fmaf(w, s_l[g][k], ll);
    }
    c_acc[k][e] = a;
    if (e == 0) {
      c_m[k] = mm;
      c_l[k] = ll;
    }
  }
  cluster.sync();
  if (cta == 0) {
    for (int idx = tid; idx < NB * HEAD_DIM; idx += BD_CA_THREADS) {
      const int k = idx / HEAD_DIM, e = idx % HEAD_DIM;
      if (k >= rows_per_utt) continue;
      float mm = -INFINITY;
      for (int c = 0; c < BD_CA_CLUSTER; ++c) mm = fmaxf(mm, *cluster.map_shared_rank(&c_m[k], c));
      float a = 0.f, ll = 0.f;
      for (int c = 0; c < BD_CA_CLUSTER; ++c) {
        const float mc = *cluster.map_shared_rank(&c_m[k], c);
        const float w = (mc == -INFINITY) ? 0.f : __expf(mc - mm);
        a = fmaf(w, *cluster.map_shared_rank(&c_acc[k][e], c), a);
        ll = fmaf(w, *cluster.map_shared_rank(&c_l[k], c), ll);
      }
      ctx[static_cast<long long>(u * rows_per_utt + k) * d + h * HEAD_DIM + e] = __float2half_rn(a / ll);
    }
  }
  cluster.sync();  // keep every CTA's shared memory alive until the leader has read it
}

// =====================================================================================================================
// cross-attention on wgmma (the default for the batched pass): persistent CTAs walk (utterance, head) items; the item's
// K and V (2 x 1500 x 64 fp16 = 384 KB) stream ONCE through a TMA ring for all rows of the utterance.
//   S^T = K Q^T : per 128-key tile, two wgmma.m64n8k16 x 4 (keys on M, the <= 8 query rows of the utterance on N), so
//                 all 128 threads of the warpgroup have softmax work even with 5 query rows; the scores of all 12 tiles
//                 stay in registers (96 per thread)
//   softmax     : one exact row maximum / row sum over the 1500 keys (shuffles + 4-way shared memory), P^T -> fp16,
//                 swizzled shared memory
//   O^T = V^T P : wgmma.m64n8k16 (A = the V tile as loaded, MN-major; head dim on M) x 8 per tile, accumulated over the
//                 12 tiles in registers; rows are scaled by 1/rowsum on the way out
// Warps 0..3 = the consumer warpgroup, warp 4 = TMA producer (ring order per item: 12 K tiles, then 12 V tiles, so the
// V tiles stream while the softmax runs).  Finished utterances are skipped.
// =====================================================================================================================
constexpr int XT_CONS = 128;
constexpr int XT_THREADS = XT_CONS + 32;
constexpr int XT_TILE = 128 * HEAD_DIM * 2;        // 16 KB: 128 keys of K or of V
constexpr int XT_STAGES = 8;
constexpr int XT_NT = T_ENC_PAD / 128;             // 12 key tiles per item
constexpr int XT_NQ = 8;                           // query rows padded to the MMA N
static_assert(MAX_BEAM <= XT_NQ, "cross-attention: one MMA column per row of an utterance");
constexpr int XT_P_TILE = XT_NQ * 128 * 2;         // 2 KB: P^T [8 rows][128 keys] = two swizzled 64-key halves
constexpr int XT_Q_BYTES = XT_NQ * HEAD_DIM * 2;   // 1 KB
constexpr int XT_OFF_P = XT_STAGES * XT_TILE;
constexpr int XT_OFF_Q = XT_OFF_P + XT_NT * XT_P_TILE;
constexpr int XT_OFF_BAR = XT_OFF_Q + 1024;
constexpr int XT_OFF_RED = XT_OFF_BAR + 2 * XT_STAGES * 8;         // [2][4 warps][8 rows] fp32: row max, row sum partials
constexpr int XT_OFF_LIVE = XT_OFF_RED + 2 * 4 * XT_NQ * 4;        // [BD_CROSS_MAX_UTT] unsigned short: live utterances
constexpr int XT_OFF_NLIVE = XT_OFF_LIVE + BD_CROSS_MAX_UTT * 2;   // int: number of live utterances
constexpr int XT_SMEM = XT_OFF_NLIVE + 4 + 1024;                   // + slack for the 1024-byte alignment of the base
static_assert(BD_CROSS_MAX_UTT <= 65536, "cross-attention: the live list holds utterance indices as unsigned short");
constexpr float XT_LOG2E = 1.4426950408889634f;

__global__ void __launch_bounds__(XT_THREADS, 1)
bd_cross_attn_tc_kernel(const __grid_constant__ CUtensorMap map_kv, const float* __restrict__ q, long long row_k0,
                        long long row_v0, const int* __restrict__ done, __half* __restrict__ ctx, int n_utt,
                        int rows_per_utt, int d, int H) {
  extern __shared__ uint8_t xt_raw[];
  const uint32_t raw_addr = smem_u32(xt_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;
  uint8_t* smem = xt_raw + (base - raw_addr);
  const uint32_t sP = base + XT_OFF_P, sQ = base + XT_OFF_Q;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + XT_OFF_BAR);
  const uint32_t bar0 = smem_u32(bars);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (XT_STAGES + s); };
  float* s_red = reinterpret_cast<float*>(smem + XT_OFF_RED);  // [2][4 warps][8 rows]: row max, row sum partials

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    for (int s = 0; s < XT_STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), XT_CONS / 32);  // one arrival per consumer warp
    }
    fence_mbar_init();
    tma_prefetch_desc(&map_kv);
  }
  // P^T and Q^T rows beyond the live query rows are zero for the whole kernel
  for (int i = threadIdx.x; i < (XT_NT * XT_P_TILE + XT_Q_BYTES) / 16; i += XT_THREADS)
    *reinterpret_cast<uint4*>(smem + XT_OFF_P + i * 16) = make_uint4(0u, 0u, 0u, 0u);
  fence_proxy_async_smem();
  __syncthreads();
  pdl_wait();  // q and the `done` flags come from the previous kernels of the chain

  // live utterances, compacted: item k of this CTA is (s_live[idx / H], idx % H) with idx = blockIdx.x + k * gridDim.x, so the
  // CTAs stay balanced whichever utterances have finished
  unsigned short* s_live = reinterpret_cast<unsigned short*>(smem + XT_OFF_LIVE);
  int* s_nlive = reinterpret_cast<int*>(smem + XT_OFF_NLIVE);
  if (threadIdx.x == 0) {
    int n = 0;
    for (int u = 0; u < n_utt; ++u)
      if (done == nullptr || done[u] == 0) s_live[n++] = static_cast<unsigned short>(u);
    *s_nlive = n;
  }
  __syncthreads();
  const int n_idx = *s_nlive * H;
  const int n_my = (static_cast<int>(blockIdx.x) < n_idx) ? (n_idx - 1 - static_cast<int>(blockIdx.x)) / static_cast<int>(gridDim.x) + 1 : 0;
  auto item_of = [&](int k) {  // -> u * H + h of this CTA's k-th item
    const int idx = blockIdx.x + k * gridDim.x;
    return static_cast<int>(s_live[idx / H]) * H + idx % H;
  };

  if (warp == XT_CONS / 32) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      unsigned unit = 0;
      auto load12 = [&](long long row0) {
        for (int j = 0; j < XT_NT; ++j, ++unit) {
          const int st = unit % XT_STAGES;
          mbar_wait(empty_bar(st), ((unit / XT_STAGES) & 1u) ^ 1u);
          mbar_arrive_expect_tx(full_bar(st), XT_TILE);
          tma_load_2d(base + st * XT_TILE, &map_kv, full_bar(st), 0, static_cast<int>(row0 + j * 128));
        }
      };
      for (int k = 0; k < n_my; ++k) {
        load12(row_k0 + static_cast<long long>(item_of(k)) * T_ENC_PAD);
        load12(row_v0 + static_cast<long long>(item_of(k)) * T_ENC_PAD);
      }
    }
    return;
  }
  // ------------------------------------------------------------ consumer warpgroup
  // accumulator fragment: M rows 16 warp + lane / 4 (+ 8), N columns (query rows) cq + {0, 1}
  const int cq = 2 * (lane & 3);
  auto cons_sync = [] { asm volatile("bar.sync 1, 128;" ::: "memory"); };
  unsigned unit = 0;
  auto take = [&]() {  // wait for the next ring unit -> its shared memory address
    const int st = unit % XT_STAGES;
    mbar_wait(full_bar(st), (unit / XT_STAGES) & 1u);
    return base + st * XT_TILE;
  };
  auto give_back = [&]() {  // this warp's MMAs on the current unit have completed
    if (lane == 0) mbar_arrive(empty_bar(unit % XT_STAGES));
    ++unit;
  };
  for (int it = 0; it < n_my; ++it) {
    const int item = item_of(it);
    const int u = item / H, h = item - u * H;
    // Q rows of the item -> fp16, pre-scaled by head_dim^-0.5 (exact), K-major 128-byte-swizzled rows
    if (threadIdx.x < rows_per_utt * 8) {
      const int r = threadIdx.x >> 3, c = threadIdx.x & 7;
      const float* qr = q + static_cast<long long>(u * rows_per_utt + r) * d + h * HEAD_DIM + c * 8;
      const float4 a0 = *reinterpret_cast<const float4*>(qr), a1 = *reinterpret_cast<const float4*>(qr + 4);
      __half2 h0 = __floats2half2_rn(a0.x * 0.125f, a0.y * 0.125f), h1 = __floats2half2_rn(a0.z * 0.125f, a0.w * 0.125f);
      __half2 h2 = __floats2half2_rn(a1.x * 0.125f, a1.y * 0.125f), h3 = __floats2half2_rn(a1.z * 0.125f, a1.w * 0.125f);
      uint4 v4;
      v4.x = *reinterpret_cast<uint32_t*>(&h0); v4.y = *reinterpret_cast<uint32_t*>(&h1);
      v4.z = *reinterpret_cast<uint32_t*>(&h2); v4.w = *reinterpret_cast<uint32_t*>(&h3);
      *reinterpret_cast<uint4*>(smem + XT_OFF_Q + r * 128 + ((c ^ (r & 7)) << 4)) = v4;
    }
    fence_proxy_async_smem();
    cons_sync();
    // S^T: sc[j][half][i]: key 128 j + 64 half + 16 warp + lane / 4 + 8 (i >> 1), query row cq + (i & 1)
    float sc[XT_NT][2][4];
    const uint64_t dq = make_desc_sw128(sQ, 1024);
#pragma unroll
    for (int j = 0; j < XT_NT; ++j) {
      const uint32_t tile = take();
      wgmma_fence();
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const uint64_t dk = make_desc_sw128(tile + hf * (XT_TILE / 2), 1024);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<XT_NQ, 0, 0>(sc[j][hf], dk + 2u * k, dq + 2u * k, k != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(sc[j][0]);
      wgmma_reg_fence(sc[j][1]);
      give_back();
    }
    // keys >= 1500 are padding rows of the window
    const int key_lo = warp * 16 + (lane >> 2);
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if ((XT_NT - 1) * 128 + hf * 64 + key_lo + 8 * (i >> 1) >= T_ENC) sc[XT_NT - 1][hf][i] = -INFINITY;
    // exact row maximum over all keys (lanes with the same lane % 4 hold the same query rows)
    float* red = s_red;
    float mx[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float m = -INFINITY;
#pragma unroll
      for (int j = 0; j < XT_NT; ++j)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) m = fmaxf(m, fmaxf(sc[j][hf][e], sc[j][hf][2 + e]));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
      if (lane < 4) red[warp * 8 + cq + e] = m;
    }
    cons_sync();
#pragma unroll
    for (int e = 0; e < 2; ++e)
      mx[e] = fmaxf(fmaxf(red[cq + e], red[8 + cq + e]), fmaxf(red[16 + cq + e], red[24 + cq + e])) * XT_LOG2E;
    // probabilities -> P^T tiles (fp16), row sums
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < XT_NT; ++j) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int e = i & 1, r = cq + e, kk = key_lo + 8 * (i >> 1);
          const __half ph = __float2half_rn(exp2f(fmaf(sc[j][hf][i], XT_LOG2E, -mx[e])));
          sum[e] += __half2float(ph);  // the sum of what the tensor core will actually multiply
          if (r < rows_per_utt)
            *reinterpret_cast<__half*>(smem + XT_OFF_P + j * XT_P_TILE + hf * 1024 + r * 128 + (((kk >> 3) ^ (r & 7)) << 4) +
                                       (kk & 7) * 2) = ph;
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float t = sum[e];
      t += __shfl_xor_sync(0xffffffffu, t, 4);
      t += __shfl_xor_sync(0xffffffffu, t, 8);
      t += __shfl_xor_sync(0xffffffffu, t, 16);
      if (lane < 4) red[32 + warp * 8 + cq + e] = t;
    }
    fence_proxy_async_smem();
    cons_sync();
    // O^T [64 dims x 8 rows]
    float o[4];
#pragma unroll 1
    for (int j = 0; j < XT_NT; ++j) {
      const uint32_t tile = take();
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint64_t dv = make_desc_sw128(tile + k * 2048, 1024);
        const uint64_t dp = make_desc_sw128(sP + j * XT_P_TILE + (k >> 2) * 1024, 1024) + 2u * (k & 3);
        wgmma_ss<XT_NQ, 1, 0>(o, dv, dp, (j | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(o);
      give_back();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = cq + (i & 1), e = key_lo + 8 * (i >> 1);
      if (r < rows_per_utt) {
        const float l = (red[32 + r] + red[40 + r]) + (red[48 + r] + red[56 + r]);
        ctx[static_cast<long long>(u * rows_per_utt + r) * d + h * HEAD_DIM + e] = __float2half_rn(o[i] / l);
      }
    }
  }
}

// =====================================================================================================================
// cross-attention for wide prefill passes (more than 8 query rows per utterance): one warpgroup CTA per (64-row query
// tile, head, utterance), the encoder attention's scheme (encoder.cu enc_attn_kernel) on the cross K/V.
//   Q            : the tile's fp32 rows -> fp16 after the exact 1/8 scale, as bd_cross_attn_tc_kernel rounds them,
//                  written K-major in the 128-byte-swizzled image; rows past the utterance's last are zero
//   S = Q K^T    : wgmma.m64n128k16 per 128-key tile, online softmax (running max / sum) on the accumulator fragment
//   O += P V     : wgmma.m64n64k16 with P as the register A operand, V as loaded (MN-major)
// Thread 0 feeds a 2-stage K/V ring with TMA.  The map is either the 128B-swizzled map over the linear K/V or a plain map
// over the persistent pass's chunk-swizzled K/V (16-byte chunk c of key t at c ^ (t & 7)): key tiles start at multiples
// of 128 keys and the stages are 1024-byte aligned, so both land as the same shared-memory image.  The tiles of one
// (head, utterance) are adjacent in the grid, so its 384 KB of K/V are read from HBM about once.  Keys >= 1500 are
// masked, and the last tile's V padding rows are zeroed in shared memory (0 x NaN would poison O).
// =====================================================================================================================
constexpr int PX_THREADS = 128;
constexpr int PX_BM = 64;
constexpr int PX_NB = T_ENC_PAD / 128;        // 12 key tiles
constexpr int PX_TILE = 128 * HEAD_DIM * 2;   // 16 KB: 128 keys of K or of V
constexpr int PX_Q_BYTES = PX_BM * HEAD_DIM * 2;
constexpr int PX_SMEM = PX_Q_BYTES + 4 * PX_TILE /*K, V x 2 stages*/ + 64 /*barriers*/ + 1024 /*alignment slack*/;
constexpr int PX_PAD0 = T_ENC - (PX_NB - 1) * 128;  // first padding row of the last tile (92)

__device__ __forceinline__ uint32_t px_pack(float a, float b) {
  __half2 v = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

__global__ void __launch_bounds__(PX_THREADS, 3)
bd_prefill_cross_attn_kernel(const __grid_constant__ CUtensorMap map_kv, const float* __restrict__ q, long long row_k0,
                             long long row_v0, __half* __restrict__ ctx, int rows_per_utt, int d, int H) {
  extern __shared__ uint8_t px_raw[];
  const uint32_t raw_addr = smem_u32(px_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;
  uint8_t* smem = px_raw + (base - raw_addr);
  const uint32_t sQ = base;
  const uint32_t sK = base + PX_Q_BYTES;
  const uint32_t sV = sK + 2 * PX_TILE;
  const uint32_t bar0 = sV + 2 * PX_TILE;
  auto kv_full = [&](int s) { return bar0 + 8u * s; };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = blockIdx.x, h = blockIdx.y, u = blockIdx.z;
  const long long item = static_cast<long long>(u) * H + h;
  const long long rk = row_k0 + item * T_ENC_PAD, rv = row_v0 + item * T_ENC_PAD;
  const int r0 = qt * PX_BM;

  if (tid == 0) {
    mbar_init(kv_full(0), 1);
    mbar_init(kv_full(1), 1);
    fence_mbar_init();
    tma_prefetch_desc(&map_kv);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // q comes from the cross-query GEMM just before

  auto load_kv = [&](int j) {
    const int st = j & 1;
    mbar_arrive_expect_tx(kv_full(st), 2 * PX_TILE);
    tma_load_2d(sK + st * PX_TILE, &map_kv, kv_full(st), 0, static_cast<int>(rk + j * 128));
    tma_load_2d(sV + st * PX_TILE, &map_kv, kv_full(st), 0, static_cast<int>(rv + j * 128));
  };
  if (tid == 0) {
    load_kv(0);
    load_kv(1);
  }
  for (int i = tid; i < PX_BM * 8; i += PX_THREADS) {
    const int r = i >> 3, c = i & 7, row = r0 + r;
    uint4 v4 = make_uint4(0u, 0u, 0u, 0u);
    if (row < rows_per_utt) {
      const float* qr = q + (static_cast<long long>(u) * rows_per_utt + row) * d + h * HEAD_DIM + c * 8;
      const float4 a0 = *reinterpret_cast<const float4*>(qr), a1 = *reinterpret_cast<const float4*>(qr + 4);
      v4.x = px_pack(a0.x * 0.125f, a0.y * 0.125f);
      v4.y = px_pack(a0.z * 0.125f, a0.w * 0.125f);
      v4.z = px_pack(a1.x * 0.125f, a1.y * 0.125f);
      v4.w = px_pack(a1.z * 0.125f, a1.w * 0.125f);
    }
    *reinterpret_cast<uint4*>(smem + r * 128 + ((c ^ (r & 7)) << 4)) = v4;
  }
  fence_proxy_async_smem();
  __syncthreads();

  // this thread's accumulator rows: 16 warp + lane / 4 and + 8; columns 8 j + 2 (lane % 4) + {0, 1}
  const int cq = 2 * (lane & 3);
  const float c = XT_LOG2E;  // (q is already scaled by head_dim^-0.5)
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float o[HEAD_DIM / 2];
#pragma unroll
  for (int i = 0; i < HEAD_DIM / 2; ++i) o[i] = 0.f;
  const uint64_t dq = make_desc_sw128(sQ, 1024);
#pragma unroll 1
  for (int j = 0; j < PX_NB; ++j) {
    const int st = j & 1;
    mbar_wait(kv_full(st), (j >> 1) & 1u);
    if (j == PX_NB - 1) {  // padding rows of V: whole 128-byte rows, so the swizzle does not matter
      for (int i = tid; i < (128 - PX_PAD0) * 8; i += PX_THREADS)
        *reinterpret_cast<uint4*>(smem + (sV - base) + st * PX_TILE + PX_PAD0 * 128 + i * 16) = make_uint4(0u, 0u, 0u, 0u);
      fence_proxy_async_smem();
      __syncthreads();
    }
    float s[64];
    const uint64_t dk = make_desc_sw128(sK + st * PX_TILE, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss<128, 0, 0>(s, dq + 2u * k, dk + 2u * k, k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(s);
    const int kv0 = j * 128;
    if (kv0 + 128 > T_ENC) {
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (kv0 + (i >> 2) * 8 + cq + (i & 1) >= T_ENC) s[i] = -INFINITY;
    }
    float alpha[2], mc[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float mx = -INFINITY;
#pragma unroll
      for (int nb = 0; nb < 16; ++nb) mx = fmaxf(mx, fmaxf(s[4 * nb + 2 * hr], s[4 * nb + 2 * hr + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[hr], mx);
      alpha[hr] = exp2f((m_run[hr] - m_new) * c);
      mc[hr] = m_new * c;
      m_run[hr] = m_new;
    }
    uint32_t pa[8][4];
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      float p[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        p[i] = __half2float(__float2half_rn(exp2f(fmaf(s[8 * kk + i], c, -mc[(i >> 1) & 1]))));
        rs[(i >> 1) & 1] += p[i];  // the sum of what the tensor core will actually multiply
      }
      pa[kk][0] = px_pack(p[0], p[1]);
      pa[kk][1] = px_pack(p[2], p[3]);
      pa[kk][2] = px_pack(p[4], p[5]);
      pa[kk][3] = px_pack(p[6], p[7]);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) l_run[hr] = l_run[hr] * alpha[hr] + rs[hr];
#pragma unroll
    for (int i = 0; i < HEAD_DIM / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) wgmma_rs<HEAD_DIM, 1>(o, pa[kk], make_desc_sw128(sV + st * PX_TILE + kk * 2048, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(o);
    __syncthreads();  // every thread's MMAs have read stage st: refill it
    if (tid == 0 && j + 2 < PX_NB) load_kv(j + 2);
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 1);
    l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 2);
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = r0 + warp * 16 + (lane >> 2) + 8 * hr;
    if (row >= rows_per_utt) continue;
    const float inv = 1.0f / l_run[hr];
    __half* out = ctx + (static_cast<long long>(u) * rows_per_utt + row) * d + h * HEAD_DIM + cq;
#pragma unroll
    for (int nb = 0; nb < HEAD_DIM / 8; ++nb)
      *reinterpret_cast<uint32_t*>(out + nb * 8) = px_pack(o[4 * nb + 2 * hr] * inv, o[4 * nb + 2 * hr + 1] * inv);
  }
}

// =====================================================================================================================
// alignment capture (Whisper.align): one CTA per (alignment head of this layer, utterance).  The item's query rows are
// rounded to fp16 after the exact 1/8 scale, as bd_cross_attn_tc_kernel feeds them to the tensor core, the scores against
// all 1500 keys stay in shared memory, and one exact fp32 row maximum / row sum gives the probabilities the decoder itself
// attends with.  Only rows at positions s0 .. s0 + n_text[u] and frames < n_frames[u] are written.
// =====================================================================================================================
constexpr int AC_THREADS = 256;
constexpr int AC_SMEM = (MAX_BEAM * HEAD_DIM + MAX_BEAM * T_ENC) * 4;  // q [8][64] + scores [8][1500]

__global__ void __launch_bounds__(AC_THREADS)
bd_align_attn_kernel(const AlignCaptureArgs a) {
  extern __shared__ float ac_smem[];
  float* s_q = ac_smem;
  float* s_p = ac_smem + MAX_BEAM * HEAD_DIM;
  __shared__ float s_red[AC_THREADS / 32][MAX_BEAM];
  __shared__ float s_stat[MAX_BEAM];
  const int u = blockIdx.y, ga = a.items[blockIdx.x];
  const int h = a.head_of[ga];
  const int rpu = a.rows_per_utt, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = a.n_text[u];
  const int* rp = a.row_pos + u * rpu;
  // uniform over the CTA: does any row of this pass land in the captured range?
  if (rp[rpu - 1] < a.s0 || rp[0] > a.s0 + n || n <= 0) return;
  for (int i = tid; i < rpu * HEAD_DIM; i += AC_THREADS) {
    const int k = i / HEAD_DIM, e = i % HEAD_DIM;
    s_q[i] = __half2float(__float2half_rn(a.q[static_cast<long long>(u * rpu + k) * a.d + h * HEAD_DIM + e] * 0.125f));
  }
  __syncthreads();
  const __half* kb = a.ck + (static_cast<long long>(u) * a.H + h) * T_ENC_PAD * HEAD_DIM;
  float mx[MAX_BEAM];
#pragma unroll
  for (int k = 0; k < MAX_BEAM; ++k) mx[k] = -INFINITY;
  for (int t = tid; t < T_ENC; t += AC_THREADS) {
    const uint4* kr = reinterpret_cast<const uint4*>(kb + static_cast<long long>(t) * HEAD_DIM);
    float acc[MAX_BEAM];
#pragma unroll
    for (int k = 0; k < MAX_BEAM; ++k) acc[k] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint4 uu = __ldg(kr + i);
      const __half2* h2 = reinterpret_cast<const __half2*>(&uu);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h2[j]);
#pragma unroll
        for (int k = 0; k < MAX_BEAM; ++k)
          if (k < rpu) {
            acc[k] = fmaf(s_q[k * HEAD_DIM + 8 * i + 2 * j], f.x, acc[k]);
            acc[k] = fmaf(s_q[k * HEAD_DIM + 8 * i + 2 * j + 1], f.y, acc[k]);
          }
      }
    }
#pragma unroll
    for (int k = 0; k < MAX_BEAM; ++k)
      if (k < rpu) {
        s_p[k * T_ENC + t] = acc[k];
        mx[k] = fmaxf(mx[k], acc[k]);
      }
  }
#pragma unroll
  for (int k = 0; k < MAX_BEAM; ++k) {
    const float m = warp_max(mx[k]);
    if (lane == 0) s_red[warp][k] = m;
  }
  __syncthreads();
  if (tid < rpu) {
    float m = -INFINITY;
    for (int w = 0; w < AC_THREADS / 32; ++w) m = fmaxf(m, s_red[w][tid]);
    s_stat[tid] = m;
  }
  __syncthreads();
  float sum[MAX_BEAM];
#pragma unroll
  for (int k = 0; k < MAX_BEAM; ++k) {
    sum[k] = 0.f;
    if (k < rpu) {
      const float m = s_stat[k];
      for (int t = tid; t < T_ENC; t += AC_THREADS) {
        const float e = expf(s_p[k * T_ENC + t] - m);
        s_p[k * T_ENC + t] = e;
        sum[k] += e;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < MAX_BEAM; ++k) {
    const float v = warp_sum(sum[k]);
    if (lane == 0) s_red[warp][k] = v;
  }
  __syncthreads();
  if (tid < rpu) {
    float v = 0.f;
    for (int w = 0; w < AC_THREADS / 32; ++w) v += s_red[w][tid];
    s_stat[tid] = v;
  }
  __syncthreads();
  const int F = a.n_frames[u];
  for (int k = 0; k < rpu; ++k) {
    const int r = rp[k] - a.s0;
    if (r < 0 || r > n) continue;
    const float l = s_stat[k];
    float* dst = a.cap + ((static_cast<long long>(u) * a.A + ga) * (a.n_max + 1) + r) * a.f_max;
    for (int f = tid; f < F; f += AC_THREADS) dst[f] = s_p[k * T_ENC + f] / l;
  }
}

template <typename Kern, typename... Args>
void bd_launch(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = pdl ? 1 : 0;
  WISB_CUDA(cudaLaunchKernelEx(&cfg, kern, args...));
}

int bd_ca_smem(int nb) { return 2 * BD_CA_KEYS * HEAD_DIM * 2 + BD_CA_GROUPS * nb * HEAD_DIM * 4; }

void cross_tc_launch(const BatchArgs& a, const BatchLayer& ly, cudaStream_t s) {
  static std::atomic<unsigned long long> once{0};
  once_per_device(once, [] {
    WISB_CUDA(cudaFuncSetAttribute(bd_cross_attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, XT_SMEM));
  });
  const int items = a.n_utt * a.H;
  const long long row_k0 = (ly.ck - a.ckv_base) / HEAD_DIM, row_v0 = (ly.cv - a.ckv_base) / HEAD_DIM;
  bd_launch(bd_cross_attn_tc_kernel, dim3(items < a.num_sms ? items : a.num_sms), dim3(XT_THREADS), XT_SMEM, s, a.pdl != 0,
            *a.ckv_map, a.q, row_k0, row_v0, a.done, a.ctx, a.n_utt, a.rows_per_utt, a.d, a.H);
}

void run_gemm_rows(const GemmPlan& plan, int rows, int pdl, cudaStream_t s) {
  GemmPlan p = plan;  // the plan is built for the buffer capacity; this pass uses the first `rows` rows
  p.M = round_up(rows, 128);
  if (p.M > plan.M) p.M = plan.M;
  p.epi.m_valid = rows;
  p.pdl = pdl;
  gemm_run(p, s);
}

}  // namespace

void embed_ln_launch(const BatchArgs& a, const float* g, const float* b, cudaStream_t s) {
  bd_launch(bd_embed_ln_kernel, dim3(cdiv(a.R, BD_LN_WARPS)), dim3(BD_LN_WARPS * 32), 0, s, a.pdl != 0, a.tokens, a.row_pos,
            a.tok_emb, a.pos_emb, g, b, a.x, a.xn, a.d, a.R);
}

void self_attn_launch(const BatchArgs& a, const BatchLayer& ly, cudaStream_t s) {
  bd_launch(bd_self_attn_kernel, dim3(cdiv(a.H, 4), a.R), dim3(128), 0, s, a.pdl != 0, a.q, ly.kcache, ly.vcache, a.row_pos,
            a.row_slot, a.indir0, a.indir1, a.flip, a.done, a.ctx, a.d, a.H, a.t_cap, a.t_ind, a.rows_per_utt, a.prefill);
}

void prefill_cross_attn_launch(const BatchArgs& a, const BatchLayer& ly, cudaStream_t s) {
  WISB_REQUIRE(a.n_utt >= 1 && a.n_utt <= 65535 && a.rows_per_utt >= 1 && a.rows_per_utt <= BD_SA_TMAX && a.H >= 1 && a.H <= 65535,
               "prefill cross-attention: 1..65535 utterances and heads, 1..448 rows per utterance");
  static std::atomic<unsigned long long> once{0};
  once_per_device(once, [] {
    WISB_CUDA(cudaFuncSetAttribute(bd_prefill_cross_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PX_SMEM));
  });
  const long long row_k0 = (ly.ck - a.ckv_base) / HEAD_DIM, row_v0 = (ly.cv - a.ckv_base) / HEAD_DIM;
  bd_launch(bd_prefill_cross_attn_kernel, dim3(cdiv(a.rows_per_utt, PX_BM), a.H, a.n_utt), dim3(PX_THREADS), PX_SMEM, s,
            a.pdl != 0, *a.ckv_map, a.q, row_k0, row_v0, a.ctx, a.rows_per_utt, a.d, a.H);
}

void cross_attn_launch(const BatchArgs& a, const BatchLayer& ly, cudaStream_t s) {
  if (a.wide || a.rows_per_utt > MAX_BEAM) {
    prefill_cross_attn_launch(a, ly, s);
    return;
  }
  WISB_REQUIRE(a.n_utt >= 1 && a.n_utt <= BD_CROSS_MAX_UTT,
               "cross-attention: 1.." + std::to_string(BD_CROSS_MAX_UTT) + " utterances in one pass, got " + std::to_string(a.n_utt));
  if (a.cross_tc) {
    cross_tc_launch(a, ly, s);
    return;
  }
  static std::atomic<unsigned long long> once{0};
  once_per_device(once, [&] {
    WISB_CUDA(cudaFuncSetAttribute(bd_cross_attn_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, bd_ca_smem(1)));
    WISB_CUDA(cudaFuncSetAttribute(bd_cross_attn_kernel<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, bd_ca_smem(5)));
    WISB_CUDA(cudaFuncSetAttribute(bd_cross_attn_kernel<MAX_BEAM>, cudaFuncAttributeMaxDynamicSharedMemorySize, bd_ca_smem(MAX_BEAM)));
  });
  dim3 grid(a.H, a.n_utt, BD_CA_CLUSTER);
  const int rpu = a.rows_per_utt;
  if (rpu == 1)
    bd_launch(bd_cross_attn_kernel<1>, grid, dim3(BD_CA_THREADS), bd_ca_smem(1), s, a.pdl != 0, a.q, ly.ck, ly.cv, a.done, a.ctx, rpu, a.d, a.H);
  else if (rpu <= 5)
    bd_launch(bd_cross_attn_kernel<5>, grid, dim3(BD_CA_THREADS), bd_ca_smem(5), s, a.pdl != 0, a.q, ly.ck, ly.cv, a.done, a.ctx, rpu, a.d, a.H);
  else
    bd_launch(bd_cross_attn_kernel<MAX_BEAM>, grid, dim3(BD_CA_THREADS), bd_ca_smem(MAX_BEAM), s, a.pdl != 0, a.q, ly.ck, ly.cv, a.done, a.ctx, rpu, a.d, a.H);
}

void resid_ln_launch(const BatchArgs& a, int n_splits, const float* bias, const float* g, const float* b, cudaStream_t s) {
  const dim3 grid(cdiv(a.R, BD_LN_WARPS)), block(BD_LN_WARPS * 32);
  const bool pdl = a.pdl != 0;
  switch (n_splits) {
    case 1: bd_launch(bd_resid_ln_kernel<1>, grid, block, 0, s, pdl, a.x, a.part, a.part_stride, bias, g, b, a.xn, a.d, a.R); break;
    case 2: bd_launch(bd_resid_ln_kernel<2>, grid, block, 0, s, pdl, a.x, a.part, a.part_stride, bias, g, b, a.xn, a.d, a.R); break;
    case 4: bd_launch(bd_resid_ln_kernel<4>, grid, block, 0, s, pdl, a.x, a.part, a.part_stride, bias, g, b, a.xn, a.d, a.R); break;
    case 8: bd_launch(bd_resid_ln_kernel<8>, grid, block, 0, s, pdl, a.x, a.part, a.part_stride, bias, g, b, a.xn, a.d, a.R); break;
    default: throw Error(1, "batched decoder pass: split-K factor must be 1, 2, 4 or 8");
  }
}

void align_capture_run(const AlignCaptureArgs& a, cudaStream_t s) {
  WISB_REQUIRE(a.rows_per_utt >= 1 && a.rows_per_utt <= MAX_BEAM, "alignment capture: 1..8 rows per utterance");
  if (a.n_items == 0 || a.n_utt == 0) return;
  static std::atomic<unsigned long long> once{0};
  once_per_device(once, [] {
    WISB_CUDA(cudaFuncSetAttribute(bd_align_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AC_SMEM));
  });
  bd_align_attn_kernel<<<dim3(a.n_items, a.n_utt), AC_THREADS, AC_SMEM, s>>>(a);
  WISB_CUDA(cudaGetLastError());
}

int batch_pass_run(const BatchArgs& a, const BatchLayer* layers, int n_layers, cudaStream_t s) {
  WISB_REQUIRE(a.R >= 1 && a.R == a.n_utt * a.rows_per_utt, "batched decoder pass: rows must be utterances x rows per utterance");
  WISB_REQUIRE(a.rows_per_utt >= 1 && (a.rows_per_utt <= MAX_BEAM || (a.prefill && a.rows_per_utt <= BD_SA_TMAX)),
               "batched decoder pass: 1..8 rows per utterance, 1..448 in a prefill pass");
  WISB_REQUIRE(a.d % 128 == 0 && a.d <= 128 * BD_LN_MAX, "batched decoder pass: d_model multiple of 128, <= 1536");
  WISB_REQUIRE(a.t_ind <= BD_SA_TMAX, "batched decoder pass: more than 448 text positions");
  struct Scope {  // brackets one kernel with the optional timing hook
    const BatchArgs& a;
    Scope(const BatchArgs& a_, int cat) : a(a_) {
      if (a.prof) a.prof(a.prof_ctx, cat, 1);
    }
    ~Scope() {
      if (a.prof) a.prof(a.prof_ctx, 0, 0);
    }
  };
  int n = 0;
  {
    Scope t(a, 2);
    embed_ln_launch(a, layers[0].ln1g, layers[0].ln1b, s);
  }
  ++n;
  auto gemm = [&](const GemmPlan& p) {
    Scope t(a, 0);
    run_gemm_rows(p, a.R, a.pdl, s);
  };
  auto ln = [&](int splits, const float* bias, const float* g, const float* b) {
    Scope t(a, 2);
    resid_ln_launch(a, splits, bias, g, b, s);
  };
  for (int i = 0; i < n_layers; ++i) {
    const BatchLayer& ly = layers[i];
    gemm(ly.qkv);
    {
      Scope t(a, 3);
      self_attn_launch(a, ly, s);
    }
    gemm(ly.o);
    ln(ly.o.k_splits, ly.ob, ly.ln2g, ly.ln2b);
    gemm(ly.cq);
    if (a.layer_hook) n += a.layer_hook(a.hook_ctx, i, s);
    {
      Scope t(a, 1);
      cross_attn_launch(a, ly, s);
    }
    gemm(ly.co);
    ln(ly.co.k_splits, ly.cob, ly.ln3g, ly.ln3b);
    gemm(ly.fc1);
    gemm(ly.fc2);
    ln(ly.fc2.k_splits, ly.fc2b, ly.next_g, ly.next_b);
    n += 11;
  }
  if (a.with_logits) {
    gemm(*a.vocab);
    ++n;
  }
  return n;
}

}  // namespace wisb
