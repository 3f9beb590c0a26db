// wgmma GEMM for sm_90a:  D[M,N] = A[M,K] . W[N,K]^T   (fp16 x fp16 -> fp32 in registers) with fused epilogues.
//
// Replaces (reference side): every dense layer CTranslate2 runs through cuBLAS `gemmEx` for
// ctranslate2.models.Whisper.generate (main.py:687-692 of the reference server; SURVEY.md section 2b rows K3,K5,K7-K9,K11).
//
// Structure (one persistent CTA per SM, 384 threads = 3 warpgroups):
//   warps 0..7  two consumer warpgroups: warpgroup g issues wgmma.m64nBNk16 (x4 per stage) for rows [64 g, 64 g + 64) of
//               the 128-row tile, accumulates in registers, then runs the bias / GELU / residual / scatter epilogues
//               (each warp stages its accumulator through shared memory, 16 rows x 64 columns at a time, so that each
//               of its 32 threads writes one row's 32 consecutive columns with vector stores)
//   warps 8..11 producer warpgroup, one thread of which issues cp.async.bulk.tensor 128x64 (A) and BNx64 (W) fp16 tiles,
//               128B swizzle, into a STAGES-deep ring; it gives most of its registers to the consumers (setmaxnreg), which
//               hold up to 128 fp32 accumulators per thread at BN = 256
// The ring keeps streaming the next tiles' operands while the consumers run an epilogue.
#include <mutex>

#include "kernels.h"
#include "ptx.cuh"

namespace wisb {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;
constexpr int GEMM_CONSUMERS = 256;                 // two warpgroups
constexpr int GEMM_THREADS = GEMM_CONSUMERS + 128;  // + producer warpgroup
// a warp's epilogue staging slice: 16 rows x two 32-column halves, fp32; row stride 66 and half offset 33 put the 32
// lanes' reads (lane = row + 16 half) in 32 different banks
constexpr int EPI_LD = 66, EPI_HALF = 33;
constexpr int EPI_BYTES = (GEMM_CONSUMERS / 32) * 16 * EPI_LD * 4;

template <int BN>
struct GemmCfg {
  static constexpr int STAGES = (BN == 256) ? 4 : (BN == 160 ? 5 : (BN == 128 ? 6 : 8));
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int SMEM_BYTES = STAGES * (A_STAGE_BYTES + B_STAGE_BYTES) + EPI_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "gemm: shared memory per block");
};

__device__ __forceinline__ void store_f16x32(__half* dst, const float (&f)[32]) {
  uint4* d4 = reinterpret_cast<uint4*>(dst);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 h0 = __floats2half2_rn(f[8 * i + 0], f[8 * i + 1]);
    __half2 h1 = __floats2half2_rn(f[8 * i + 2], f[8 * i + 3]);
    __half2 h2 = __floats2half2_rn(f[8 * i + 4], f[8 * i + 5]);
    __half2 h3 = __floats2half2_rn(f[8 * i + 6], f[8 * i + 7]);
    uint4 u;
    u.x = *reinterpret_cast<uint32_t*>(&h0);
    u.y = *reinterpret_cast<uint32_t*>(&h1);
    u.z = *reinterpret_cast<uint32_t*>(&h2);
    u.w = *reinterpret_cast<uint32_t*>(&h3);
    d4[i] = u;
  }
}

// One thread owns one output row and 32 consecutive columns [col0, col0+32).
__device__ __forceinline__ void epilogue_chunk(const GemmEpi& e, int row, int col0, const float (&v)[32], int split) {
  float f[32];
  if (e.bias != nullptr) {
    const float4* b4 = reinterpret_cast<const float4*>(e.bias + col0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float4 b = __ldg(b4 + i);
      f[4 * i + 0] = v[4 * i + 0] + b.x;
      f[4 * i + 1] = v[4 * i + 1] + b.y;
      f[4 * i + 2] = v[4 * i + 2] + b.z;
      f[4 * i + 3] = v[4 * i + 3] + b.w;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 32; ++i) f[i] = v[i];
  }
  switch (e.mode) {
    case EPI_F16_GELU:
#pragma unroll
      for (int i = 0; i < 32; ++i) f[i] = gelu_erf(f[i]);
      // fallthrough
    case EPI_F16:
      store_f16x32(reinterpret_cast<__half*>(e.out) + static_cast<long long>(row) * e.ldo + col0, f);
      break;
    case EPI_RESID_F32: {
      float4* o4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(e.out) + static_cast<long long>(row) * e.ldo + col0);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float4 o = o4[i];
        o.x += f[4 * i + 0];
        o.y += f[4 * i + 1];
        o.z += f[4 * i + 2];
        o.w += f[4 * i + 3];
        o4[i] = o;
      }
      break;
    }
    case EPI_CONV2: {
      const int t = row % T_ENC_PAD;
      float4* o4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(e.out) + static_cast<long long>(row) * e.ldo + col0);
      if (t < T_ENC) {
        const float4* p4 = reinterpret_cast<const float4*>(e.pos + static_cast<long long>(t) * e.ldo + col0);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float4 p = __ldg(p4 + i);
          o4[i] = make_float4(gelu_erf(f[4 * i + 0]) + p.x, gelu_erf(f[4 * i + 1]) + p.y, gelu_erf(f[4 * i + 2]) + p.z,
                              gelu_erf(f[4 * i + 3]) + p.w);
        }
      } else {  // padding rows of the window: keep them exactly zero
#pragma unroll
        for (int i = 0; i < 8; ++i) o4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      break;
    }
    case EPI_CROSSKV: {
      // col -> (layer, k|v, head, e); row -> (b, t); out [layer][kv][b][head][1536][64]
      const int two_d = 2 * e.d_model;
      const int layer = col0 / two_d;
      const int within = col0 - layer * two_d;
      const int kv = within / e.d_model;
      const int c = within - kv * e.d_model;
      const int head = c >> 6, e0 = c & 63;
      const int b = row / T_ENC_PAD, t = row - b * T_ENC_PAD;
      long long idx = ((((static_cast<long long>(layer) * 2 + kv) * e.batch + e.batch_off + b) * e.n_heads + head) * T_ENC_PAD + t) * 64;
      if (e.kv_swizzle) {
        // persistent warp-MMA decoder pass: the 16-byte chunks of a key's 128-byte row are XOR-swizzled by the key index, so
        // that the bulk-copied rows are ldmatrix-conflict-free in shared memory (unswizzled: 8-way bank conflicts per
        // ldmatrix.x4).  The batched pass reads the linear layout through a TMA swizzle instead.
        uint4* row = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(e.out) + idx);
        const int c0 = e0 >> 3;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          __half2 h0 = __floats2half2_rn(f[8 * i + 0], f[8 * i + 1]);
          __half2 h1 = __floats2half2_rn(f[8 * i + 2], f[8 * i + 3]);
          __half2 h2 = __floats2half2_rn(f[8 * i + 4], f[8 * i + 5]);
          __half2 h3 = __floats2half2_rn(f[8 * i + 6], f[8 * i + 7]);
          uint4 u;
          u.x = *reinterpret_cast<uint32_t*>(&h0);
          u.y = *reinterpret_cast<uint32_t*>(&h1);
          u.z = *reinterpret_cast<uint32_t*>(&h2);
          u.w = *reinterpret_cast<uint32_t*>(&h3);
          row[(c0 + i) ^ (t & 7)] = u;
        }
      } else {
        store_f16x32(reinterpret_cast<__half*>(e.out) + idx + e0, f);
      }
      break;
    }
    case EPI_QKV_VT: {
      if (col0 < 2 * e.d_model) {
        store_f16x32(reinterpret_cast<__half*>(e.out) + static_cast<long long>(row) * e.ldo + col0, f);
      } else {  // V part, transposed per head: vt[((b*H + head)*64 + e)][t]
        const int c = col0 - 2 * e.d_model;
        const int head = c >> 6, e0 = c & 63;
        const int b = row / T_ENC_PAD, t = row - b * T_ENC_PAD;
        __half* vt = reinterpret_cast<__half*>(e.aux) +
                     (static_cast<long long>(b * e.n_heads + head) * 64 + e0) * T_ENC_PAD + t;
#pragma unroll
        for (int i = 0; i < 32; ++i) vt[static_cast<long long>(i) * T_ENC_PAD] = __float2half_rn(f[i]);
      }
      break;
    }
    case EPI_F32: {
      float4* o4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(e.out) + split * e.split_stride +
                                             static_cast<long long>(row) * e.ldo + col0);
#pragma unroll
      for (int i = 0; i < 8; ++i) o4[i] = make_float4(f[4 * i + 0], f[4 * i + 1], f[4 * i + 2], f[4 * i + 3]);
      break;
    }
    case EPI_DEC_QKV: {
      const int d = e.d_model;
      if (col0 < d) {  // query: fp32 [rows, d]
        float4* o4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(e.out) + static_cast<long long>(row) * e.ldo + col0);
#pragma unroll
        for (int i = 0; i < 8; ++i) o4[i] = make_float4(f[4 * i + 0], f[4 * i + 1], f[4 * i + 2], f[4 * i + 3]);
      } else {         // key / value of this row's position, straight into the self-attention cache
        const bool is_v = col0 >= 2 * d;
        const int c = col0 - (is_v ? 2 * d : d);
        const long long at = (static_cast<long long>(__ldg(e.row_slot + row)) * e.t_cap + __ldg(e.row_pos + row)) * d + c;
        store_f16x32(reinterpret_cast<__half*>(is_v ? e.aux2 : e.aux) + at, f);
      }
      break;
    }
    default:
      break;
  }
}

// kMC: launched as clusters of 2 CTAs that own vertically adjacent M tiles of the same N tile; each CTA fetches half of
// the W tile and TMA-multicasts it to both, which cuts the L2->SM operand traffic per MMA from (128+BN) to (128+BN/2) rows.
// A stage is free again once the consumers of BOTH CTAs have read it (the peer multicasts into it too).
template <int BN, bool kMC>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int M, int N, int K,
               int a_wrap, int k_splits, const GemmEpi epi) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;  // 128B-swizzle atoms need 1024-byte alignment
  uint8_t* smem = smem_raw + (base - raw_addr);
  const uint32_t smem_a0 = base;
  const uint32_t smem_b0 = base + STAGES * A_STAGE_BYTES;
  float* epi_stage = reinterpret_cast<float*>(smem + STAGES * (A_STAGE_BYTES + Cfg::B_STAGE_BYTES));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * (A_STAGE_BYTES + Cfg::B_STAGE_BYTES) + EPI_BYTES);
  const uint32_t bar0 = smem_u32(bars);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();  // (no-op unless the next kernel was launched with the programmatic-serialization attribute)
  const int n_tiles = (N + BN - 1) / BN;
  // split-K: a work item is (tile, K range); its partial goes to its own output slab (EPI_F32) and is summed by the
  // consumer kernel in a fixed order (deterministic, no atomics)
  const int k_blocks = K / BK / k_splits;
  // work items: single tiles, or (kMC) vertical tile pairs handled by a 2-CTA cluster (rank r takes M tile 2 * pair + r)
  const uint32_t crank = kMC ? cluster_ctarank() : 0u;
  const int first_unit = kMC ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);
  const int unit_stride = kMC ? static_cast<int>(gridDim.x >> 1) : static_cast<int>(gridDim.x);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), (GEMM_CONSUMERS / 128) * (kMC ? 2 : 1));  // one arrival per consumer warpgroup (and CTA)
    }
    fence_mbar_init();
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
  }
  __syncthreads();
  if (kMC) cluster_sync_all();  // peer barriers are initialised before any multicast copy / remote arrival can reach them
  pdl_wait();  // everything above overlapped the previous kernel's tail; its results are visible from here on
  // rows actually present (device-side count, e.g. the rows of the utterances still decoding): whole M tiles beyond it
  // are skipped by both roles alike
  int m_tiles = M / BM;
  if (epi.m_dyn != nullptr) {
    const int mt = (*epi.m_dyn + BM - 1) / BM;
    if (mt < m_tiles) m_tiles = mt;
  }
  if (kMC) m_tiles = (m_tiles + 1) & ~1;  // pairs of M tiles (the tensor map always covers an even number of tiles here)
  const int m_units = kMC ? m_tiles / 2 : m_tiles;
  const int total_tiles = m_units * n_tiles * k_splits;
  auto unit_split = [&](int unit) { return unit % k_splits; };
  auto unit_m0 = [&](int unit) { return (((unit / k_splits) % m_units) * (kMC ? 2 : 1) + static_cast<int>(crank)) * BM; };
  auto unit_n0 = [&](int unit) { return ((unit / k_splits) / m_units) * BN; };

  if (warp >= GEMM_CONSUMERS / 32) {
    // ------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (warp == GEMM_CONSUMERS / 32 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = first_unit; tile < total_tiles; tile += unit_stride) {
        const int m0 = unit_m0(tile);
        const int n0 = unit_n0(tile);
        const int kb0 = unit_split(tile) * k_blocks;
        for (int kbl = 0; kbl < k_blocks; ++kbl) {
          const int kb = kb0 + kbl;
          mbar_wait(empty_bar(stage), phase ^ 1u);
          mbar_arrive_expect_tx(full_bar(stage), A_STAGE_BYTES + Cfg::B_STAGE_BYTES);
          // a_wrap > 0: logical A row r = [phys row r | first K - a_wrap columns of phys row r + 1]  (conv2 view)
          int ka = kb * BK, ra = m0;
          if (a_wrap > 0 && ka >= a_wrap) {
            ka -= a_wrap;
            ra += 1;
          }
          tma_load_2d(smem_a0 + stage * A_STAGE_BYTES, &map_a, full_bar(stage), ka, ra);
          if (kMC) {  // my half of the W tile, delivered to both CTAs (the peer delivers the other half)
            tma_load_2d_mcast(smem_b0 + stage * Cfg::B_STAGE_BYTES + crank * (Cfg::B_STAGE_BYTES / 2), &map_b, full_bar(stage),
                              kb * BK, n0 + static_cast<int>(crank) * (BN / 2), 0x3);
          } else {
            tma_load_2d(smem_b0 + stage * Cfg::B_STAGE_BYTES, &map_b, full_bar(stage), kb * BK, n0);
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers: MMA + epilogue
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;                          // rows [64 wg, 64 wg + 64) of the tile
    const bool signaller = (threadIdx.x & 127) == 0;   // one arrival per warpgroup on the empty barriers
    auto release = [&](int s) {
      if (signaller) {
        if (kMC) {
          mbar_arrive_cluster(empty_bar(s), 0);
          mbar_arrive_cluster(empty_bar(s), 1);
        } else {
          mbar_arrive(empty_bar(s));
        }
      }
    };
    float* stg = epi_stage + warp * 16 * EPI_LD;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = first_unit; tile < total_tiles; tile += unit_stride) {
      const int m0 = unit_m0(tile);
      const int n0 = unit_n0(tile);
      const int split = unit_split(tile);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint64_t da = make_desc_sw128(smem_a0 + stage * A_STAGE_BYTES + wg * (A_STAGE_BYTES / 2), 1024);
        const uint64_t db = make_desc_sw128(smem_b0 + stage * Cfg::B_STAGE_BYTES, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          // advance 16 fp16 = 32 bytes inside the 128-byte swizzle row: +2 in the (addr >> 4) field
          wgmma_ss<BN, 0, 0>(acc, da + 2u * k, db + 2u * k, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous stage's MMAs are done: hand its buffers back to the producer
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc);
      if (prev >= 0) release(prev);
      // epilogue: pairs of 32-column slices of the warp's 16 rows through shared memory; lane (r + 16 h) then owns
      // row r's 32 columns of slice 2 p + h, so every lane writes one row chunk per pair
      const int row = m0 + wg * 64 + (warp & 3) * 16 + (lane & 15);
      const int hl = lane >> 4;
      const int r0 = lane >> 2, c0 = (lane & 3) * 2;
#pragma unroll
      for (int p = 0; p < (BN / 32 + 1) / 2; ++p) {
        if (n0 + 64 * p >= epi.n_valid) break;  // warp-uniform
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int c = 2 * p + h;
          if (c < BN / 32) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int nb = 4 * c + j;
              stg[r0 * EPI_LD + h * EPI_HALF + j * 8 + c0] = acc[4 * nb + 0];
              stg[r0 * EPI_LD + h * EPI_HALF + j * 8 + c0 + 1] = acc[4 * nb + 1];
              stg[(r0 + 8) * EPI_LD + h * EPI_HALF + j * 8 + c0] = acc[4 * nb + 2];
              stg[(r0 + 8) * EPI_LD + h * EPI_HALF + j * 8 + c0 + 1] = acc[4 * nb + 3];
            }
          }
        }
        __syncwarp();
        const int col0 = n0 + (2 * p + hl) * 32;
        if (2 * p + hl < BN / 32 && col0 < epi.n_valid && row < epi.m_valid) {
          float v[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = stg[(lane & 15) * EPI_LD + hl * EPI_HALF + i];
          epilogue_chunk(epi, row, col0, v, split);
        }
        __syncwarp();
      }
    }
  }
  __syncthreads();
  if (kMC) cluster_sync_all();  // the peer may still be multicasting into / arriving on this CTA's shared memory
}

// ------------------------------------------------------------------ SIMT cross-check
__global__ void gemm_ref_kernel(const __half* __restrict__ a, long long lda, const __half* __restrict__ w, float* c, int M,
                                int N, int K) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = blockIdx.y;
  if (n >= N || m >= M) return;
  const __half* ar = a + static_cast<long long>(m) * lda;
  const __half* wr = w + static_cast<long long>(n) * K;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc = fmaf(__half2float(ar[k]), __half2float(wr[k]), acc);
  c[static_cast<long long>(m) * N + n] = acc;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  if (!fn) throw Error(2, "cuTensorMapEncodeTiled is not available from the CUDA driver");
  return fn;
}

}  // namespace

// 2-D fp16 tensor map: inner dimension `cols` (contiguous), `rows` rows of stride `ld` elements, 128B swizzle
void make_tmap_f16_2d(CUtensorMap* map, const void* ptr, long long cols, long long rows, long long ld, int box_cols,
                      int box_rows) {
  make_tmap_f16_2d_swizzle(map, ptr, cols, rows, ld, box_cols, box_rows, true);
}

void make_tmap_f16_2d_swizzle(CUtensorMap* map, const void* ptr, long long cols, long long rows, long long ld,
                              int box_cols, int box_rows, bool swizzle_128b) {
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode_fn()(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE,
                               swizzle_128b ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw Error(2, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string(static_cast<int>(r)));
}

void gemm_plan(GemmPlan& p, const __half* a, long long lda, const __half* w, int M, int N, int K, const GemmEpi& epi,
               int num_sms, int force_bn, int a_wrap, int k_splits) {
  WISB_REQUIRE(M > 0 && M % BM == 0, "gemm: M must be a positive multiple of 128");
  WISB_REQUIRE(K > 0 && K % BK == 0, "gemm: K must be a positive multiple of 64");
  WISB_REQUIRE(N > 0 && N % 32 == 0, "gemm: N must be a positive multiple of 32");
  WISB_REQUIRE((lda * 2) % 16 == 0 && (reinterpret_cast<uintptr_t>(a) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0,
               "gemm: operands must be 16-byte aligned");
  WISB_REQUIRE(k_splits >= 1 && (K / BK) % k_splits == 0, "gemm: K blocks must divide evenly over the K splits");
  WISB_REQUIRE(k_splits == 1 || (epi.mode == EPI_F32 && epi.split_stride > 0), "gemm: split-K needs the EPI_F32 partial epilogue");
  p.M = M;
  p.N = N;
  p.K = K;
  p.k_splits = k_splits;
  p.epi = epi;
  if (p.epi.m_valid <= 0) p.epi.m_valid = M;
  if (p.epi.n_valid <= 0) p.epi.n_valid = N;
  const bool no_mcast = force_bn < 0;
  int bn = force_bn < 0 ? -force_bn : force_bn;
  if (bn == 0) {
    // wave quantisation on `num_sms` CTAs dominates at one window (M = 1536): pick the tile width with the fewest
    // (waves x tile cost); e.g. N = 3840 -> 160 (288 tiles = 1.95 waves) instead of 256 (180 tiles = 1.22 -> 2 waves)
    long long best = -1;
    for (int cand : {256, 160, 128}) {
      if (N % cand != 0) continue;
      const long long t = static_cast<long long>(M / BM) * (N / cand);
      const long long cost = ((t + num_sms - 1) / num_sms) * (cand + 48);
      if (best < 0 || cost < best) {
        best = cost;
        bn = cand;
      }
    }
    if (bn == 0) bn = 128;
  }
  WISB_REQUIRE(bn == 64 || bn == 128 || bn == 160 || bn == 256, "gemm: BN must be 64, 128, 160 or 256");
  p.BN = bn;
  const int tiles = (M / BM) * ((N + bn - 1) / bn) * k_splits;
  // 2-CTA clusters with multicast W tiles whenever the M tiles pair up and N tiles are whole
  p.mcast = (!no_mcast && (M / BM) % 2 == 0 && N % bn == 0 && a_wrap == 0 && num_sms >= 2) ? 1 : 0;
  if (p.mcast) {
    const int units = tiles / 2, clusters = num_sms / 2;
    p.grid = 2 * (units < clusters ? units : clusters);
  } else {
    p.grid = tiles < num_sms ? tiles : num_sms;
  }
  p.a_wrap = a_wrap;
  if (a_wrap > 0) {
    WISB_REQUIRE(a_wrap % BK == 0 && lda == a_wrap && K > a_wrap && K - a_wrap <= a_wrap, "gemm: bad a_wrap");
    make_tmap_f16_2d(&p.map_a, a, a_wrap, M + 1, lda, BK, BM);
  } else {
    make_tmap_f16_2d(&p.map_a, a, K, M, lda, BK, BM);
  }
  make_tmap_f16_2d(&p.map_b, w, K, N, K, BK, p.mcast ? bn / 2 : bn);
}

template <int BN, bool kMC>
void gemm_launch(const GemmPlan& p, cudaStream_t stream) {
  static std::atomic<unsigned long long> once{0};
  once_per_device(once, [] {
    WISB_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, kMC>, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<BN>::SMEM_BYTES));
  });
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(p.grid);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = GemmCfg<BN>::SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kMC ? 2 : 1;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = p.pdl ? 2 : 1;
  WISB_CUDA(cudaLaunchKernelEx(&cfg, gemm_tc_kernel<BN, kMC>, p.map_a, p.map_b, p.M, p.N, p.K, p.a_wrap, p.k_splits, p.epi));
}

void gemm_run(const GemmPlan& p, cudaStream_t stream) {
  if (p.BN == 64) {
    if (p.mcast) gemm_launch<64, true>(p, stream); else gemm_launch<64, false>(p, stream);
  } else if (p.BN == 256) {
    if (p.mcast) gemm_launch<256, true>(p, stream); else gemm_launch<256, false>(p, stream);
  } else if (p.BN == 160) {
    if (p.mcast) gemm_launch<160, true>(p, stream); else gemm_launch<160, false>(p, stream);
  } else {
    if (p.mcast) gemm_launch<128, true>(p, stream); else gemm_launch<128, false>(p, stream);
  }
}

void gemm_ref_run(const __half* a, long long lda, const __half* w, float* c, int M, int N, int K, cudaStream_t stream) {
  dim3 grid(cdiv(N, 128), M);
  gemm_ref_kernel<<<grid, 128, 0, stream>>>(a, lda, w, c, M, N, K);
  WISB_CUDA(cudaGetLastError());
}

}  // namespace wisb
