// Whisper encoder pieces that are not plain GEMMs: conv1 stem, LayerNorm, non-causal self-attention.
//
// Replaces (reference side) the encoder half of ctranslate2.models.Whisper.generate
// (main.py:687-692 of the reference server; SURVEY.md section 2b rows K2, K4, K6).  Architecture per
// [HF] modeling_whisper.py:567-568,619-625 (conv stem), :361-415 (encoder layer).
#include <mutex>

#include "kernels.h"
#include "ptx.cuh"

namespace wisb {

void make_tmap_f16_2d(CUtensorMap* map, const void* ptr, long long cols, long long rows, long long ld, int box_cols,
                      int box_rows);

namespace {

// =====================================================================================================================
// conv1: Conv1d(80 -> d, k=3, pad=1) + GELU.  1.8 GFLOP per window (0.1 % of the encoder): fp32 FMA, smem tiled.
// Output row layout (fp16 [B, 3072, d]): row 0 = zeros (left pad), rows 1..3000 = frames, rows 3001.. = zeros, so that
// conv2 (k=3, stride 2, pad 1) is a plain GEMM whose A row t' is the 3*d contiguous values starting at row 2*t'.
// =====================================================================================================================
constexpr int C1_FT = 64;   // frames per CTA
constexpr int C1_CT = 64;   // output channels per CTA
constexpr int C1_K = 3 * N_MELS;
constexpr int C1_SMEM = (N_MELS * (C1_FT + 2) + C1_K * (C1_CT + 1)) * 4;

__global__ void __launch_bounds__(256)
conv1_gelu_kernel(const float* __restrict__ mel, const __half* __restrict__ w, const float* __restrict__ bias,
                  __half* __restrict__ h1, int d) {
  extern __shared__ float c1_smem[];
  float (*xm)[C1_FT + 2] = reinterpret_cast<float (*)[C1_FT + 2]>(c1_smem);
  float (*wt)[C1_CT + 1] = reinterpret_cast<float (*)[C1_CT + 1]>(c1_smem + N_MELS * (C1_FT + 2));
  const int b = blockIdx.z;
  const int f0 = blockIdx.x * C1_FT;
  const int c0 = blockIdx.y * C1_CT;
  const int tid = threadIdx.x;
  const float* melb = mel + static_cast<long long>(b) * N_MELS * N_FRAMES;
  for (int i = tid; i < N_MELS * (C1_FT + 2); i += 256) {
    const int ci = i / (C1_FT + 2), fl = i % (C1_FT + 2);
    const int f = f0 + fl - 1;
    xm[ci][fl] = (f >= 0 && f < N_FRAMES) ? melb[ci * N_FRAMES + f] : 0.f;
  }
  for (int i = tid; i < C1_CT * C1_K; i += 256) {
    const int co = i / C1_K, kk = i % C1_K;
    wt[kk][co] = __half2float(w[static_cast<long long>(c0 + co) * C1_K + kk]);
  }
  __syncthreads();
  const int tc = tid % 16;  // 4 channels each
  const int tf = tid / 16;  // 4 frames each
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int kk = 0; kk < C1_K; ++kk) {
    const int k = kk / N_MELS, ci = kk - k * N_MELS;
    float a[4], bb[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = xm[ci][tf * 4 + i + k];
#pragma unroll
    for (int j = 0; j < 4; ++j) bb[j] = wt[kk][tc * 4 + j];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int f = f0 + tf * 4 + i;
    if (f >= N_FRAMES) continue;
    __half* o = h1 + (static_cast<long long>(b) * H1_ROWS + 1 + f) * d + c0 + tc * 4;
    __half2 v0 = __floats2half2_rn(gelu_erf(acc[i][0] + bias[c0 + tc * 4 + 0]), gelu_erf(acc[i][1] + bias[c0 + tc * 4 + 1]));
    __half2 v1 = __floats2half2_rn(gelu_erf(acc[i][2] + bias[c0 + tc * 4 + 2]), gelu_erf(acc[i][3] + bias[c0 + tc * 4 + 3]));
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&v0);
    u.y = *reinterpret_cast<uint32_t*>(&v1);
    *reinterpret_cast<uint2*>(o) = u;
  }
}

// =====================================================================================================================
// LayerNorm: one warp per row, fp32 in, fp16 out (feeds the next GEMM's A operand). eps = 1e-5, biased variance.
// =====================================================================================================================
constexpr int LN_MAX_IT = 12;  // d <= 1536

__global__ void __launch_bounds__(256)
layernorm_f32_to_f16_kernel(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ b,
                            __half* __restrict__ y, int rows, int d) {
  pdl_launch_dependents();  // (programmatic dependent launch: the next kernel's prologue overlaps this one)
  pdl_wait();               // the producer of x has completed
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int iters = d / 128;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<long long>(row) * d);
  float4 v[LN_MAX_IT];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_IT; ++i)
    if (i < iters) {
      v[i] = xr[i * 32 + lane];
      s += v[i].x + v[i].y + v[i].z + v[i].w;
    }
  const float mean = warp_sum(s) / d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_IT; ++i)
    if (i < iters) {
      const float a0 = v[i].x - mean, a1 = v[i].y - mean, a2 = v[i].z - mean, a3 = v[i].w - mean;
      q += a0 * a0 + a1 * a1 + a2 * a2 + a3 * a3;
    }
  const float rstd = rsqrtf(warp_sum(q) / d + 1e-5f);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const float4* b4 = reinterpret_cast<const float4*>(b);
  uint2* yr = reinterpret_cast<uint2*>(y + static_cast<long long>(row) * d);
#pragma unroll
  for (int i = 0; i < LN_MAX_IT; ++i)
    if (i < iters) {
      const float4 gg = __ldg(g4 + i * 32 + lane), bb = __ldg(b4 + i * 32 + lane);
      __half2 h0 = __floats2half2_rn((v[i].x - mean) * rstd * gg.x + bb.x, (v[i].y - mean) * rstd * gg.y + bb.y);
      __half2 h1 = __floats2half2_rn((v[i].z - mean) * rstd * gg.z + bb.z, (v[i].w - mean) * rstd * gg.w + bb.w);
      uint2 u;
      u.x = *reinterpret_cast<uint32_t*>(&h0);
      u.y = *reinterpret_cast<uint32_t*>(&h1);
      yr[i * 32 + lane] = u;
    }
}

// =====================================================================================================================
// Encoder self-attention on wgmma: one CTA = one warpgroup per (64-query tile, head, window), 3 CTAs per SM.
//   S = Q K^T          : wgmma.m64n128k16 (4 instr per 128-key block), fp32 in registers
//   softmax            : online (running max / sum per query row) on the accumulator fragment, exp2; the probabilities
//                        become the fp16 A operand in registers without a trip through shared memory
//   O += P V_j         : wgmma.m64n64k16 with A from registers (8 instr per block), O rescaled in registers
// Thread 0 also feeds the 2-stage K/V ring with TMA.  Keys >= 1500 (padding rows of the 1536-row window) are masked.
// V operand: kVMN = true  -> V tile as loaded [kv][dh] (MN-major B descriptor)
//            kVMN = false -> pre-transposed Vt [dh][kv] written by the QKV GEMM epilogue (K-major B descriptor)
// =====================================================================================================================
constexpr int AT_THREADS = 128;
constexpr int AT_BM = 64, AT_BN = 128;
constexpr int AT_NB = T_ENC_PAD / AT_BN;  // 12 key blocks
constexpr int AT_TILE = 128 * 64 * 2;     // 16 KB: 128 keys of K or of V
constexpr int AT_Q_BYTES = AT_BM * 64 * 2;
constexpr int AT_SMEM = AT_Q_BYTES + 4 * AT_TILE /*K, V x 2 stages*/ + 64 /*barriers*/ + 1024 /*alignment slack*/;

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <bool kVMN>
__global__ void __launch_bounds__(AT_THREADS, 3)
enc_attn_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                const __grid_constant__ CUtensorMap map_v, __half* __restrict__ ctx, int d, int H) {
  extern __shared__ uint8_t at_raw[];
  const uint32_t raw_addr = smem_u32(at_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;
  const uint32_t sQ = base;
  const uint32_t sK = base + AT_Q_BYTES;
  const uint32_t sV = sK + 2 * AT_TILE;
  const uint32_t bar0 = sV + 2 * AT_TILE;
  const uint32_t q_full = bar0;
  auto kv_full = [&](int s) { return bar0 + 8u * (1 + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int row0 = b * T_ENC_PAD + qt * AT_BM;

  if (tid == 0) {
    mbar_init(q_full, 1);
    mbar_init(kv_full(0), 1);
    mbar_init(kv_full(1), 1);
    fence_mbar_init();
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // barriers and descriptors were set up under the QKV GEMM's tail; its output is visible from here on

  auto load_kv = [&](int j) {
    const int st = j & 1;
    mbar_arrive_expect_tx(kv_full(st), 2 * AT_TILE);
    tma_load_2d(sK + st * AT_TILE, &map_k, kv_full(st), d + h * HEAD_DIM, b * T_ENC_PAD + j * AT_BN);
    if (kVMN) {
      tma_load_2d(sV + st * AT_TILE, &map_v, kv_full(st), 2 * d + h * HEAD_DIM, b * T_ENC_PAD + j * AT_BN);
    } else {
      // Vt viewed as [B*H*64 rows, 1536 cols]; two 64x64 halves of the key block
      tma_load_2d(sV + st * AT_TILE, &map_v, kv_full(st), j * AT_BN, (b * H + h) * HEAD_DIM);
      tma_load_2d(sV + st * AT_TILE + AT_TILE / 2, &map_v, kv_full(st), j * AT_BN + 64, (b * H + h) * HEAD_DIM);
    }
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(q_full, AT_Q_BYTES);
    tma_load_2d(sQ, &map_q, q_full, h * HEAD_DIM, row0);
    load_kv(0);
    load_kv(1);
  }

  // this thread's accumulator rows: r0 = 16 warp + lane / 4 and r0 + 8; columns 8 j + 2 (lane % 4) + {0, 1}
  const int cq = 2 * (lane & 3);
  const float c = 0.125f * 1.4426950408889634f;  // dh^-0.5 * log2(e)
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float o[HEAD_DIM / 2];
#pragma unroll
  for (int i = 0; i < HEAD_DIM / 2; ++i) o[i] = 0.f;
  const uint64_t dq = make_desc_sw128(sQ, 1024);
  mbar_wait(q_full, 0);
#pragma unroll 1
  for (int j = 0; j < AT_NB; ++j) {
    const int st = j & 1;
    mbar_wait(kv_full(st), (j >> 1) & 1u);
    float s[AT_BN / 2];
    const uint64_t dk = make_desc_sw128(sK + st * AT_TILE, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss<AT_BN, 0, 0>(s, dq + 2u * k, dk + 2u * k, k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(s);
    const int kv0 = j * AT_BN;
    if (kv0 + AT_BN > T_ENC) {
#pragma unroll
      for (int i = 0; i < AT_BN / 2; ++i)
        if (kv0 + (i >> 2) * 8 + cq + (i & 1) >= T_ENC) s[i] = -INFINITY;
    }
    float alpha[2], mc[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float mx = -INFINITY;
#pragma unroll
      for (int nb = 0; nb < AT_BN / 8; ++nb) mx = fmaxf(mx, fmaxf(s[4 * nb + 2 * hr], s[4 * nb + 2 * hr + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[hr], mx);
      alpha[hr] = exp2f((m_run[hr] - m_new) * c);
      mc[hr] = m_new * c;
      m_run[hr] = m_new;
    }
    uint32_t pa[AT_BN / 16][4];
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < AT_BN / 16; ++kk) {
      float p[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        p[i] = exp2f(fmaf(s[8 * kk + i], c, -mc[(i >> 1) & 1]));
        rs[(i >> 1) & 1] += p[i];
      }
      pa[kk][0] = pack_half2(p[0], p[1]);
      pa[kk][1] = pack_half2(p[2], p[3]);
      pa[kk][2] = pack_half2(p[4], p[5]);
      pa[kk][3] = pack_half2(p[6], p[7]);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) l_run[hr] = l_run[hr] * alpha[hr] + rs[hr];
#pragma unroll
    for (int i = 0; i < HEAD_DIM / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AT_BN / 16; ++kk) {
      uint64_t dv;
      if (kVMN)
        dv = make_desc_sw128(sV + st * AT_TILE + kk * 2048, 1024);
      else
        dv = make_desc_sw128(sV + st * AT_TILE + (kk >> 2) * (AT_TILE / 2), 1024) + 2u * (kk & 3);
      wgmma_rs<HEAD_DIM, kVMN ? 1 : 0>(o, pa[kk], dv, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(o);
    __syncthreads();  // every thread's MMAs have read stage st: refill it
    if (tid == 0 && j + 2 < AT_NB) load_kv(j + 2);
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 1);
    l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 2);
  }
  const float inv[2] = {1.0f / l_run[0], 1.0f / l_run[1]};
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int r = warp * 16 + (lane >> 2) + 8 * hr;
    __half* out = ctx + static_cast<long long>(row0 + r) * d + h * HEAD_DIM + cq;
#pragma unroll
    for (int nb = 0; nb < HEAD_DIM / 8; ++nb)
      *reinterpret_cast<uint32_t*>(out + nb * 8) = pack_half2(o[4 * nb + 2 * hr] * inv[hr], o[4 * nb + 2 * hr + 1] * inv[hr]);
  }
}

// SIMT cross-check (diagnostics / tests only): one thread per query row, online softmax in fp32
__global__ void __launch_bounds__(128)
enc_attn_ref_kernel(const __half* __restrict__ qkv, __half* __restrict__ ctx, int d) {
  const int b = blockIdx.z, h = blockIdx.y;
  const int t = blockIdx.x * 128 + threadIdx.x;
  const long long ld = 3LL * d;
  const __half* base = qkv + static_cast<long long>(b) * T_ENC_PAD * ld;
  float q[HEAD_DIM], acc[HEAD_DIM];
  for (int e = 0; e < HEAD_DIM; ++e) {
    q[e] = __half2float(base[t * ld + h * HEAD_DIM + e]);
    acc[e] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  for (int k = 0; k < T_ENC; ++k) {
    const __half* kr = base + k * ld + d + h * HEAD_DIM;
    float s = 0.f;
    for (int e = 0; e < HEAD_DIM; ++e) s = fmaf(q[e], __half2float(kr[e]), s);
    s *= 0.125f;
    const float mn = fmaxf(m, s);
    const float a = __expf(m - mn), p = __expf(s - mn);
    const __half* vr = base + k * ld + 2 * d + h * HEAD_DIM;
    for (int e = 0; e < HEAD_DIM; ++e) acc[e] = acc[e] * a + p * __half2float(vr[e]);
    l = l * a + p;
    m = mn;
  }
  __half* o = ctx + (static_cast<long long>(b) * T_ENC_PAD + t) * d + h * HEAD_DIM;
  for (int e = 0; e < HEAD_DIM; ++e) o[e] = __float2half_rn(acc[e] / l);
}

}  // namespace

void conv1_gelu_run(const float* mel, const __half* w, const float* bias, __half* h1, int B, int d, cudaStream_t stream) {
  WISB_REQUIRE(d % C1_CT == 0, "conv1: d_model must be a multiple of 64");
  static std::atomic<unsigned long long> once{0};
  once_per_device(once, [] {
    WISB_CUDA(cudaFuncSetAttribute(conv1_gelu_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C1_SMEM));
  });
  dim3 grid(cdiv(N_FRAMES, C1_FT), d / C1_CT, B);
  conv1_gelu_kernel<<<grid, 256, C1_SMEM, stream>>>(mel, w, bias, h1, d);
  WISB_CUDA(cudaGetLastError());
}

void layernorm_f32_to_f16_run(const float* x, const float* g, const float* b, __half* y, int rows, int d,
                              cudaStream_t stream, bool pdl) {
  WISB_REQUIRE(d % 128 == 0 && d <= 128 * LN_MAX_IT, "layernorm: d_model must be a multiple of 128, <= 1536");
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cdiv(rows, 8));
  cfg.blockDim = dim3(256);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  WISB_CUDA(cudaLaunchKernelEx(&cfg, layernorm_f32_to_f16_kernel, x, g, b, y, rows, d));
}

void enc_attn_plan(AttnPlan& p, const __half* qkv, const __half* vt, __half* ctx, int B, int d, int H, bool v_mn_major) {
  p.B = B;
  p.d = d;
  p.H = H;
  p.ctx = ctx;
  p.v_mn_major = v_mn_major;
  const long long rows = static_cast<long long>(B) * T_ENC_PAD;
  make_tmap_f16_2d(&p.map_q, qkv, 3LL * d, rows, 3LL * d, 64, AT_BM);
  make_tmap_f16_2d(&p.map_k, qkv, 3LL * d, rows, 3LL * d, 64, 128);
  if (v_mn_major)
    make_tmap_f16_2d(&p.map_v, qkv, 3LL * d, rows, 3LL * d, 64, 128);
  else
    make_tmap_f16_2d(&p.map_v, vt, T_ENC_PAD, static_cast<long long>(B) * H * HEAD_DIM, T_ENC_PAD, 64, 64);
}

void enc_attn_run(const AttnPlan& p, cudaStream_t stream) {
  static std::atomic<unsigned long long> once{0};
  once_per_device(once, [] {
    WISB_CUDA(cudaFuncSetAttribute(enc_attn_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, AT_SMEM));
    WISB_CUDA(cudaFuncSetAttribute(enc_attn_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AT_SMEM));
  });
  dim3 grid(T_ENC_PAD / AT_BM, p.H, p.B);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(AT_THREADS);
  cfg.dynamicSmemBytes = AT_SMEM;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = p.pdl ? 1 : 0;
  if (p.v_mn_major)
    WISB_CUDA(cudaLaunchKernelEx(&cfg, enc_attn_kernel<true>, p.map_q, p.map_k, p.map_v, p.ctx, p.d, p.H));
  else
    WISB_CUDA(cudaLaunchKernelEx(&cfg, enc_attn_kernel<false>, p.map_q, p.map_k, p.map_v, p.ctx, p.d, p.H));
}

void enc_attn_ref_run(const __half* qkv, __half* ctx, int B, int d, int H, cudaStream_t stream) {
  dim3 grid(T_ENC_PAD / 128, H, B);
  enc_attn_ref_kernel<<<grid, 128, 0, stream>>>(qkv, ctx, d);
  WISB_CUDA(cudaGetLastError());
}

}  // namespace wisb
