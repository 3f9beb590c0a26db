// Decoder step kernels for a handful of rows (utterances x beams <= 16): the HBM-bandwidth-bound part of
// ctranslate2.models.Whisper.generate (main.py:687-692; SURVEY.md section 8a row A10).
// Architecture per [HF] modeling_whisper.py:417-508 (decoder layer), :650-700 (embeddings), :966-971 (tied projection).
//
// Activations stay fp32 end to end here (weights fp16 -> fp32 on the fly, fp32 FMA): with <= 16 rows the step is bound by
// streaming the 1.8 GB of decoder weights, so the extra precision is free and keeps the arg-max decisions close to the
// fp32 oracle.  Every kernel reads the current position from DecState so a single captured CUDA graph serves all steps.
#include <cooperative_groups.h>

#include <mutex>

#include "decoder.cuh"
#include "ptx.cuh"

namespace cg = cooperative_groups;

namespace wisb {

namespace {

// =====================================================================================================================
// Skinny GEMM for <= 16 rows: out[R, N] = f(LN?(x)[R, K] . W[N, K]^T + bias), one pass over the weights.
//
// A CTA of 4 warps owns 16 consecutive output columns per task (warp w: columns 4w..4w+3) and walks K in chunks.
// Thread 0 is the TMA producer: cp.async.bulk copies of the 16 weight-row chunks (and of the activations / LayerNorm
// parameters) into shared memory, mbarrier complete_tx, a 2-stage ring one (task, chunk) unit ahead of the compute.
// Everything the math touches is therefore in shared memory, the compute loop is small and rolled (instruction
// footprint stays in the I-cache) and the bytes in flight are set by the ring, not by registers.
// Programmatic dependent launch: the weight / LayerNorm-parameter copies are issued BEFORE griddepcontrol.wait, i.e.
// while the previous kernel of the decoder chain is still running, so launch latency and HBM latency of the weight
// stream overlap the predecessor instead of adding up 260 times per decoder pass.
// LayerNorm is folded into the same pass:
//     LN(x) . w = rstd * (sum_k x_k g_k w_k  -  mean * sum_k g_k w_k) + sum_k b_k w_k
// with mean / rstd from the row sums each warp accumulates on the way (a warp sees every k of its columns).
// =====================================================================================================================
constexpr int GV_WARPS = 4;
constexpr int GV_C = 4;
constexpr int GV_COLS = GV_WARPS * GV_C;  // 16 columns per CTA task

// in: lane l holds v[0..31]; out: v[0] of lane l = sum over all lanes of their v[l]   (31 shuffles instead of 160)
__device__ __forceinline__ float warp_transpose_reduce(float (&v)[32], int lane) {
#pragma unroll
  for (int off = 16, n = 32; off >= 1; off >>= 1, n >>= 1) {
    const bool up = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      if (i < n / 2) {
        const float send = up ? v[i] : v[i + n / 2];
        const float keep = up ? v[i + n / 2] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
      }
    }
  }
  return v[0];
}

struct GemvSmem {
  int n_chunks, kc;          // K split
  int off_gb, off_x, off_ring, stage_bytes, w_bytes, total;
};
__host__ __device__ inline GemvSmem gemv_smem_layout(int R, int K, bool ln) {
  GemvSmem L;
  L.n_chunks = (K > 1536) ? 4 : 1;
  L.kc = K / L.n_chunks;
  int off = 128;  // barriers
  L.off_gb = off;
  if (ln) off += 2 * K * 4;
  L.off_x = off;
  if (L.n_chunks == 1) off += R * K * 4;
  off = (off + 127) & ~127;
  L.off_ring = off;
  L.w_bytes = GV_COLS * L.kc * 2;
  L.stage_bytes = L.w_bytes + (L.n_chunks > 1 ? R * L.kc * 4 : 0);
  L.stage_bytes = (L.stage_bytes + 127) & ~127;
  L.total = off + 2 * L.stage_bytes;
  return L;
}

template <int NR, bool LN>
__global__ void __launch_bounds__(GV_WARPS * 32)
gemv_kernel(const GemvArgs a) {
  constexpr int C = GV_C;
  extern __shared__ __align__(128) uint8_t gv_smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int R = a.R, K = a.K;
  const GemvSmem L = gemv_smem_layout(R, K, LN);
  const uint32_t sbase = smem_u32(gv_smem);
  const uint32_t bar_full0 = sbase, bar_empty0 = sbase + 16, bar_x = sbase + 32, bar_gb = sbase + 40;
  const float* s_g = reinterpret_cast<const float*>(gv_smem + L.off_gb);
  const float* s_b = s_g + K;
  const int n_tasks = (a.N + GV_COLS - 1) / GV_COLS;
  const int my_tasks = (static_cast<int>(blockIdx.x) < n_tasks) ? (n_tasks - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const int n_units = my_tasks * L.n_chunks;

  auto unit_task = [&](int unit) { return static_cast<int>(blockIdx.x) + (unit / L.n_chunks) * static_cast<int>(gridDim.x); };
  auto issue_w = [&](int unit, bool arrive_now, uint32_t extra_bytes) {  // thread 0 only
    const int task = unit_task(unit), chunk = unit % L.n_chunks, st = unit & 1;
    int rows = a.N - task * GV_COLS;
    rows = rows > GV_COLS ? GV_COLS : rows;
    const uint32_t bytes = static_cast<uint32_t>(rows * L.kc * 2);
    if (arrive_now)
      mbar_arrive_expect_tx(bar_full0 + 8 * st, bytes + extra_bytes);
    else
      mbar_expect_tx(bar_full0 + 8 * st, bytes);
    const uint32_t dst = sbase + L.off_ring + st * L.stage_bytes;
    for (int c = 0; c < rows; ++c)
      bulk_load_1d(dst + c * L.kc * 2, a.w + static_cast<long long>(task * GV_COLS + c) * K + chunk * L.kc,
                   static_cast<uint32_t>(L.kc * 2), bar_full0 + 8 * st);
  };
  auto issue_xchunk = [&](int unit) {  // thread 0 only; x chunk [R, kc] of a multi-chunk K
    const int chunk = unit % L.n_chunks, st = unit & 1;
    const uint32_t dst = sbase + L.off_ring + st * L.stage_bytes + L.w_bytes;
    for (int r = 0; r < R; ++r)
      bulk_load_1d(dst + r * L.kc * 4, a.x + static_cast<long long>(r) * K + chunk * L.kc, static_cast<uint32_t>(L.kc * 4),
                   bar_full0 + 8 * st);
  };
  const uint32_t xchunk_bytes = (L.n_chunks > 1) ? static_cast<uint32_t>(R * L.kc * 4) : 0u;

  if (tid == 0) {
    mbar_init(bar_full0, 1);
    mbar_init(bar_full0 + 8, 1);
    mbar_init(bar_empty0, GV_WARPS);
    mbar_init(bar_empty0 + 8, GV_WARPS);
    mbar_init(bar_x, 1);
    mbar_init(bar_gb, 1);
    fence_mbar_init();
    // static data first: it does not depend on the previous kernel
    if (n_units > 0) issue_w(0, /*arrive_now=*/false, 0);
    if (LN) {
      mbar_arrive_expect_tx(bar_gb, static_cast<uint32_t>(2 * K * 4));
      bulk_load_1d(sbase + L.off_gb, a.ln_g, static_cast<uint32_t>(K * 4), bar_gb);
      bulk_load_1d(sbase + L.off_gb + K * 4, a.ln_b, static_cast<uint32_t>(K * 4), bar_gb);
    }
  }
  pdl_launch_dependents();
  pdl_wait();  // activations written by the previous kernel are visible from here on
  if (tid == 0 && n_units > 0) {
    if (L.n_chunks == 1) {
      mbar_arrive_expect_tx(bar_x, static_cast<uint32_t>(R * K * 4));
      bulk_load_1d(sbase + L.off_x, a.x, static_cast<uint32_t>(R * K * 4), bar_x);
      mbar_arrive_expect_tx(bar_full0, 0);  // completes the arrival for unit 0 (bytes were announced above)
    } else {
      mbar_arrive_expect_tx(bar_full0, xchunk_bytes);
      issue_xchunk(0);
    }
  }
  __syncthreads();  // barrier inits visible to every thread
  if (n_units == 0) return;
  if (L.n_chunks == 1) mbar_wait(bar_x, 0);
  if (LN) mbar_wait(bar_gb, 0);

  float acc[C][NR], s2[C], s3[C], sx[NR], sxx[NR];
  for (int unit = 0; unit < n_units; ++unit) {
    const int chunk = unit % L.n_chunks, task = unit_task(unit), st = unit & 1;
    if (chunk == 0) {
#pragma unroll
      for (int c = 0; c < C; ++c) {
        s2[c] = s3[c] = 0.f;
#pragma unroll
        for (int r = 0; r < NR; ++r) acc[c][r] = 0.f;
      }
#pragma unroll
      for (int r = 0; r < NR; ++r) sx[r] = sxx[r] = 0.f;
    }
    if (tid == 0 && unit + 1 < n_units) {
      const int nst = (unit + 1) & 1;
      if (unit >= 1) mbar_wait(bar_empty0 + 8 * nst, ((unit - 1) >> 1) & 1u);  // all warps left that stage
      fence_proxy_async_smem();
      issue_w(unit + 1, /*arrive_now=*/true, xchunk_bytes);
      if (L.n_chunks > 1) issue_xchunk(unit + 1);
    }
    mbar_wait(bar_full0 + 8 * st, (unit >> 1) & 1u);
    const uint8_t* stage = gv_smem + L.off_ring + st * L.stage_bytes;
    const uint8_t* wst = stage + (warp * C) * L.kc * 2;
    const float* xs = (L.n_chunks == 1) ? reinterpret_cast<const float*>(gv_smem + L.off_x)
                                        : reinterpret_cast<const float*>(stage + L.w_bytes);
    const int xld = (L.n_chunks == 1) ? K : L.kc;
    const int kbase = chunk * L.kc;
#pragma unroll 1
    for (int v = lane; v < L.kc / 8; v += 32) {
      float wf[C][8];
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const uint4 u = *reinterpret_cast<const uint4*>(wst + c * L.kc * 2 + v * 16);
        const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __half22float2(h2[i]);
          wf[c][2 * i] = f.x;
          wf[c][2 * i + 1] = f.y;
        }
      }
      float g[8];
      if (LN) {
        const float4 g0 = *reinterpret_cast<const float4*>(s_g + kbase + v * 8), g1 = *reinterpret_cast<const float4*>(s_g + kbase + v * 8 + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(s_b + kbase + v * 8), b1 = *reinterpret_cast<const float4*>(s_b + kbase + v * 8 + 4);
        g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w; g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int c = 0; c < C; ++c)
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            s2[c] = fmaf(g[i], wf[c][i], s2[c]);
            s3[c] = fmaf(bb[i], wf[c][i], s3[c]);
          }
      }
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        if (r < R) {
          const float* xp = xs + r * xld + ((L.n_chunks == 1) ? kbase : 0) + v * 8;
          const float4 x0 = *reinterpret_cast<const float4*>(xp), x1 = *reinterpret_cast<const float4*>(xp + 4);
          float xv[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
          if (LN) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              sx[r] += xv[i];
              sxx[r] = fmaf(xv[i], xv[i], sxx[r]);
              xv[i] *= g[i];
            }
          }
#pragma unroll
          for (int i = 0; i < 8; ++i)  // k-element outermost: C independent chains per row are interleaved
#pragma unroll
            for (int c = 0; c < C; ++c) acc[c][r] = fmaf(xv[i], wf[c][i], acc[c][r]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty0 + 8 * st);  // this warp is done with the stage
    if (chunk != L.n_chunks - 1) continue;

    // ---- task complete: transpose-reduce over the warp; lane (c * NR + r) finishes output (r, n0 + c)
    const int n0 = task * GV_COLS + warp * C;
    float red[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) red[i] = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c)
#pragma unroll
      for (int r = 0; r < NR; ++r) red[c * NR + r] = acc[c][r];
    float v = warp_transpose_reduce(red, lane);
    float vs2 = 0.f, vs3 = 0.f, vsx = 0.f, vsxx = 0.f;
    if (LN) {
      // lanes [0,C): s2, [C,2C): s3 ; second pass lanes [0,NR): sum x, [16,16+NR): sum x^2
#pragma unroll
      for (int i = 0; i < 32; ++i) red[i] = 0.f;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        red[c] = s2[c];
        red[C + c] = s3[c];
      }
      const float t23 = warp_transpose_reduce(red, lane);
#pragma unroll
      for (int i = 0; i < 32; ++i) red[i] = 0.f;
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        red[r] = sx[r];
        red[16 + r] = sxx[r];
      }
      const float txx = warp_transpose_reduce(red, lane);
      const int oc = (lane < C * NR) ? lane / NR : 0, orow = (lane < C * NR) ? lane % NR : 0;
      vs2 = __shfl_sync(0xffffffffu, t23, oc);
      vs3 = __shfl_sync(0xffffffffu, t23, C + oc);
      vsx = __shfl_sync(0xffffffffu, txx, orow);
      vsxx = __shfl_sync(0xffffffffu, txx, 16 + orow);
    }
    if (lane < C * NR) {
      const int c = lane / NR, r = lane % NR;
      const int n = n0 + c;
      if (r < R && n < a.N) {
        if (LN) {
          const float mean = vsx / K;
          const float var = fmaxf(vsxx / K - mean * mean, 0.f);
          v = rsqrtf(var + 1e-5f) * (v - mean * vs2) + vs3;
        }
        if (a.bias != nullptr) v += a.bias[n];
        switch (a.epi) {
          case GV_STORE:
            a.out[static_cast<long long>(r) * a.ldo + n] = v;
            break;
          case GV_RESID:
            a.out[static_cast<long long>(r) * a.ldo + n] += v;
            break;
          case GV_GELU:
            a.out[static_cast<long long>(r) * a.ldo + n] = gelu_erf(v);
            break;
          case GV_QKV: {
            const int d = a.d_model;
            if (n < d) {
              a.out[static_cast<long long>(r) * a.ldo + n] = v;
            } else {
              const int pos = a.st->pos;
              __half* cache = (n < 2 * d) ? a.kcache : a.vcache;
              const int e = (n < 2 * d) ? n - d : n - 2 * d;
              cache[(static_cast<long long>(r) * a.t_max + pos) * d + e] = __float2half_rn(v);
            }
            break;
          }
          default:
            break;
        }
      }
    }
  }
}

__global__ void dec_embed_kernel(const int* __restrict__ tokens, const __half* __restrict__ tok_emb,
                                 const float* __restrict__ pos_emb, float* __restrict__ x, int d, const DecState* st) {
  pdl_launch_dependents();
  pdl_wait();
  const int r = blockIdx.x;
  const int pos = st->pos;
  const __half* e = tok_emb + static_cast<long long>(tokens[r]) * d;
  const float* p = pos_emb + static_cast<long long>(pos) * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) x[static_cast<long long>(r) * d + i] = __half2float(e[i]) + p[i];
}

// =====================================================================================================================
// self-attention over the cache: one warp per (row, head); keys t <= pos; position t of row r is stored in slot
// indir[r][t] for t < pos and in slot r for t == pos (written by this step's QKV kernel).
// =====================================================================================================================
constexpr int SA_TMAX = 448;

__global__ void __launch_bounds__(128)
dec_self_attn_kernel(const float* __restrict__ q, const __half* __restrict__ kcache, const __half* __restrict__ vcache,
                     const int* __restrict__ indir0, const int* __restrict__ indir1, const int* __restrict__ flip,
                     float* __restrict__ ctx, int d, int H, int t_max, const DecState* st) {
  __shared__ float s_p[4][SA_TMAX];
  __shared__ int s_slot[4][SA_TMAX];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x * 4 + warp;
  const int r = blockIdx.y;
  pdl_launch_dependents();
  pdl_wait();
  if (h >= H) return;
  const int pos = st->pos;
  const int* indir = (*flip ? indir1 : indir0) + static_cast<long long>(r) * t_max;
  const float* qr = q + static_cast<long long>(r) * d + h * HEAD_DIM;
  float qv[HEAD_DIM];
#pragma unroll
  for (int i = 0; i < HEAD_DIM / 4; ++i) {
    const float4 v = *reinterpret_cast<const float4*>(qr + 4 * i);
    qv[4 * i] = v.x; qv[4 * i + 1] = v.y; qv[4 * i + 2] = v.z; qv[4 * i + 3] = v.w;
  }
  float mx = -INFINITY;
  for (int t = lane; t <= pos; t += 32) {
    const int slot = (t == pos) ? r : indir[t];
    s_slot[warp][t] = slot;
    const uint4* kr = reinterpret_cast<const uint4*>(kcache + (static_cast<long long>(slot) * t_max + t) * d + h * HEAD_DIM);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint4 u = kr[i];
      const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h2[j]);
        s = fmaf(qv[8 * i + 2 * j], f.x, s);
        s = fmaf(qv[8 * i + 2 * j + 1], f.y, s);
      }
    }
    s *= 0.125f;
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
    const __half2 v = *reinterpret_cast<const __half2*>(vcache + (static_cast<long long>(s_slot[warp][t]) * t_max + t) * d +
                                                        h * HEAD_DIM + 2 * lane);
    const float2 f = __half22float2(v);
    o0 = fmaf(p, f.x, o0);
    o1 = fmaf(p, f.y, o1);
  }
  const float inv = 1.0f / sum;
  float2* o = reinterpret_cast<float2*>(ctx + static_cast<long long>(r) * d + h * HEAD_DIM + 2 * lane);
  *o = make_float2(o0 * inv, o1 * inv);
}

// =====================================================================================================================
// cross-attention: one cluster of 8 CTAs per (head, utterance); CTA c owns keys [192 c, 192 c + 192) of the 1536-row
// padded window (keys >= 1500 masked).  Inside a CTA, groups of 8 lanes walk keys with an online softmax for all
// `beam` rows at once (K/V are read once for every beam), partials are merged through shared memory, and the 8 CTAs
// merge through distributed shared memory -- no extra kernel, no global scratch.
// =====================================================================================================================
constexpr int CA_CLUSTER = 8;
constexpr int CA_KEYS = T_ENC_PAD / CA_CLUSTER;  // 192
constexpr int CA_THREADS = 128;
constexpr int CA_GROUPS = CA_THREADS / 8;        // 16 groups of 8 lanes; 12 keys each

template <int NB>
__global__ void __cluster_dims__(1, 1, CA_CLUSTER) __launch_bounds__(CA_THREADS)
dec_cross_attn_kernel(const float* __restrict__ q, const __half* __restrict__ kmat, const __half* __restrict__ vmat,
                      float* __restrict__ ctx, int beam, int d, int H) {
  // dynamic smem: [K tile 192 x 64 fp16 | V tile 192 x 64 fp16 | per-group partial accumulators]
  extern __shared__ __align__(128) uint8_t ca_smem[];
  __half* sK = reinterpret_cast<__half*>(ca_smem);
  __half* sV = sK + CA_KEYS * HEAD_DIM;
  float (*s_acc)[NB][HEAD_DIM] = reinterpret_cast<float (*)[NB][HEAD_DIM]>(ca_smem + 2 * CA_KEYS * HEAD_DIM * 2);
  __shared__ float s_m[CA_GROUPS][NB], s_l[CA_GROUPS][NB];
  __shared__ float c_acc[NB][HEAD_DIM];  // this CTA's merged partial (read by the cluster leader through DSMEM)
  __shared__ float c_m[NB], c_l[NB];
  __shared__ uint64_t s_bar;
  cg::cluster_group cluster = cg::this_cluster();
  const int h = blockIdx.x, u = blockIdx.y, cta = blockIdx.z;
  const int tid = threadIdx.x;
  const int grp = tid >> 3, gl = tid & 7;  // lane gl of group grp owns dims [8 gl, 8 gl + 8)
  const long long head_off = (static_cast<long long>(u) * H + h) * T_ENC_PAD * HEAD_DIM;
  const int t_begin = cta * CA_KEYS;
  // one elected thread streams this CTA's 192 keys and values (2 x 24 KB, contiguous) into shared memory with TMA
  const uint32_t bar = smem_u32(&s_bar);
  if (tid == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(bar, 2u * CA_KEYS * HEAD_DIM * 2u);
    bulk_load_1d(smem_u32(sK), kmat + head_off + static_cast<long long>(t_begin) * HEAD_DIM, CA_KEYS * HEAD_DIM * 2, bar);
    bulk_load_1d(smem_u32(sV), vmat + head_off + static_cast<long long>(t_begin) * HEAD_DIM, CA_KEYS * HEAD_DIM * 2, bar);
  }
  pdl_launch_dependents();
  pdl_wait();  // the encoder K/V above are static during decoding; q comes from the previous kernel

  float qv[NB][8];
#pragma unroll
  for (int k = 0; k < NB; ++k) {
    if (k < beam) {
      const float* qr = q + static_cast<long long>(u * beam + k) * d + h * HEAD_DIM + gl * 8;
      const float4 a0 = *reinterpret_cast<const float4*>(qr), a1 = *reinterpret_cast<const float4*>(qr + 4);
      qv[k][0] = a0.x; qv[k][1] = a0.y; qv[k][2] = a0.z; qv[k][3] = a0.w;
      qv[k][4] = a1.x; qv[k][5] = a1.y; qv[k][6] = a1.z; qv[k][7] = a1.w;
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
  for (int tl = grp; tl < CA_KEYS; tl += CA_GROUPS) {
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
      s *= 0.125f;
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
  for (int idx = tid; idx < NB * HEAD_DIM; idx += CA_THREADS) {
    const int k = idx / HEAD_DIM, e = idx % HEAD_DIM;
    float mm = -INFINITY;
    for (int g = 0; g < CA_GROUPS; ++g) mm = fmaxf(mm, s_m[g][k]);
    float a = 0.f, ll = 0.f;
    for (int g = 0; g < CA_GROUPS; ++g) {
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
    for (int idx = tid; idx < NB * HEAD_DIM; idx += CA_THREADS) {
      const int k = idx / HEAD_DIM, e = idx % HEAD_DIM;
      if (k >= beam) continue;
      float mm = -INFINITY;
      for (int c = 0; c < CA_CLUSTER; ++c) mm = fmaxf(mm, *cluster.map_shared_rank(&c_m[k], c));
      float a = 0.f, ll = 0.f;
      for (int c = 0; c < CA_CLUSTER; ++c) {
        const float mc = *cluster.map_shared_rank(&c_m[k], c);
        const float w = (mc == -INFINITY) ? 0.f : __expf(mc - mm);
        a = fmaf(w, *cluster.map_shared_rank(&c_acc[k][e], c), a);
        ll = fmaf(w, *cluster.map_shared_rank(&c_l[k], c), ll);
      }
      ctx[static_cast<long long>(u * beam + k) * d + h * HEAD_DIM + e] = a / ll;
    }
  }
  cluster.sync();  // keep every CTA's shared memory alive until the leader has read it
}

// launch with the programmatic-stream-serialization attribute (PDL); kernels call griddepcontrol.wait themselves
template <typename Kern, typename... Args>
void launch_pdl(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool cluster8, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[2];
  int n = 0;
  attrs[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[n].val.programmaticStreamSerializationAllowed = 1;
  ++n;
  (void)cluster8;
  cfg.attrs = attrs;
  cfg.numAttrs = n;
  WISB_CUDA(cudaLaunchKernelEx(&cfg, kern, args...));
}

template <int NR, bool LN>
void gemv_launch(const GemvArgs& a, int num_sms, cudaStream_t stream) {
  static_assert(GV_C * NR <= 32 && NR <= 16, "one lane per output");
  const GemvSmem L = gemv_smem_layout(a.R, a.K, LN);
  WISB_REQUIRE(L.total <= 220 * 1024, "gemv: activations do not fit in shared memory");
  static std::atomic<int> max_set[64];  // per device (zero-initialised): largest size configured so far
  int dev = 0;
  WISB_CUDA(cudaGetDevice(&dev));
  if (L.total > max_set[dev & 63].load()) {
    WISB_CUDA(cudaFuncSetAttribute(gemv_kernel<NR, LN>, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total));
    max_set[dev & 63].store(L.total);
  }
  const int tasks = cdiv(a.N, GV_COLS);
  const int per_sm = (220 * 1024) / (L.total + 1024) > 0 ? (220 * 1024) / (L.total + 1024) : 1;
  int grid = tasks;
  const int cap = per_sm * num_sms;
  if (grid > cap) grid = cap;
  launch_pdl(gemv_kernel<NR, LN>, dim3(grid), dim3(GV_WARPS * 32), static_cast<size_t>(L.total), stream, false, a);
}

}  // namespace

void gemv_run(const GemvArgs& a, cudaStream_t stream) {
  WISB_REQUIRE(a.K % 32 == 0 && a.R >= 1 && a.R <= 8, "gemv: bad shape");
  WISB_REQUIRE((reinterpret_cast<uintptr_t>(a.w) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.x) & 15) == 0, "gemv: operands must be 16-byte aligned");
  WISB_REQUIRE(a.ln_g == nullptr || a.K <= 1536, "gemv: LayerNorm prologue needs K <= 1536");
  static std::atomic<int> sms[64];  // per device
  int dev = 0;
  WISB_CUDA(cudaGetDevice(&dev));
  int num_sms = sms[dev & 63].load();
  if (num_sms == 0) {
    WISB_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    sms[dev & 63].store(num_sms);
  }
  const bool ln = a.ln_g != nullptr;
  if (a.R <= 2) {
    if (ln) gemv_launch<2, true>(a, num_sms, stream); else gemv_launch<2, false>(a, num_sms, stream);
  } else if (a.R <= 5) {
    if (ln) gemv_launch<5, true>(a, num_sms, stream); else gemv_launch<5, false>(a, num_sms, stream);
  } else {
    if (ln) gemv_launch<8, true>(a, num_sms, stream); else gemv_launch<8, false>(a, num_sms, stream);
  }
}

void dec_embed_run(const int* tokens, const __half* tok_emb, const float* pos_emb, float* x, int R, int d,
                   const DecState* st, cudaStream_t stream) {
  launch_pdl(dec_embed_kernel, dim3(R), dim3(256), 0, stream, false, tokens, tok_emb, pos_emb, x, d, st);
}

void dec_self_attn_run(const float* q, const __half* kcache, const __half* vcache, const int* indir0, const int* indir1,
                       const int* flip, float* ctx, int R, int d, int H, int t_max, const DecState* st,
                       cudaStream_t stream) {
  WISB_REQUIRE(t_max <= SA_TMAX, "self-attention: t_max > 448");
  dim3 grid(cdiv(H, 4), R);
  launch_pdl(dec_self_attn_kernel, grid, dim3(128), 0, stream, false, q, kcache, vcache, indir0, indir1, flip, ctx, d, H,
             t_max, st);
}

void dec_cross_attn_run(const float* q, const __half* k, const __half* v, float* ctx, int n_utt, int beam, int d, int H,
                        cudaStream_t stream) {
  WISB_REQUIRE(beam >= 1 && beam <= MAX_BEAM, "cross-attention: beam out of range");
  dim3 grid(H, n_utt, CA_CLUSTER);
  auto smem_for = [](int nb) { return 2 * CA_KEYS * HEAD_DIM * 2 + CA_GROUPS * nb * HEAD_DIM * 4; };
  static std::atomic<unsigned long long> once{0};
  once_per_device(once, [&] {
    WISB_CUDA(cudaFuncSetAttribute(dec_cross_attn_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_for(1)));
    WISB_CUDA(cudaFuncSetAttribute(dec_cross_attn_kernel<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_for(5)));
    WISB_CUDA(cudaFuncSetAttribute(dec_cross_attn_kernel<MAX_BEAM>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_for(MAX_BEAM)));
  });
  if (beam == 1)
    launch_pdl(dec_cross_attn_kernel<1>, grid, dim3(CA_THREADS), smem_for(1), stream, true, q, k, v, ctx, beam, d, H);
  else if (beam <= 5)
    launch_pdl(dec_cross_attn_kernel<5>, grid, dim3(CA_THREADS), smem_for(5), stream, true, q, k, v, ctx, beam, d, H);
  else
    launch_pdl(dec_cross_attn_kernel<MAX_BEAM>, grid, dim3(CA_THREADS), smem_for(MAX_BEAM), stream, true, q, k, v, ctx, beam, d, H);
}

}  // namespace wisb
