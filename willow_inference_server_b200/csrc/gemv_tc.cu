// Skinny GEMV on wgmma for <= 8 activation rows: out[R, N] = x[R, K] . W[N, K]^T (+ bias), W fp16 streamed once.
//
// A diagnostic kernel behind wisb_debug_gemv_tc, so that the arithmetic and the cost of a tensor-core GEMV at decoder
// sizes can be checked in isolation (the persistent decoder pass, decoder_mega.cu, uses the warp-level mma.sync instead).
//
// Swap-AB: the CTA's weight rows are the MMA's M dimension, the activation rows its N dimension:
//   A = W tile   [64 weight rows x 64 k]  K-major, 128-byte swizzle, straight from a 2-D TMA box (64 x rows_box)
//   B = x (fp16) [8 rows x 64 k]          K-major, 128-byte swizzle, written once by the consumer warpgroup
//   D            [64 x 8]                 fp32 in the warpgroup's registers
// wgmma.m64n8k16: the reduction over K happens in the tensor core; a CTA owns ceil(N / gridDim.x) weight rows in groups
// of 64.  The MMA always reads 64 rows = 8 swizzle atoms; a CTA that owns fewer rows lets it read whatever follows in
// shared memory (those output rows are never looked at), so no padding is ever streamed from HBM.
#include "decoder.cuh"
#include "ptx.cuh"

namespace wisb {

namespace {

constexpr int GT_CONS = 128;               // one consumer warpgroup
constexpr int GT_THREADS = GT_CONS + 32;   // + producer warp (lane 0 only)
constexpr int GT_STAGE = 36864;
constexpr int GT_NSTAGE = 2;
constexpr int GT_B_BYTES = 80 * 1024;      // x as fp16: K / 64 blocks of 1 KB (K <= 5120)
constexpr int GT_OFF_B = GT_NSTAGE * GT_STAGE + 8192;  // (+ 8 KB the MMA may read past the last stage)
constexpr int GT_OFF_BAR = GT_OFF_B + GT_B_BYTES;
constexpr int GT_SMEM = GT_OFF_BAR + 256 + 1024;

__device__ __forceinline__ void gt_cons_sync() { asm volatile("bar.sync 1, %0;" ::"n"(GT_CONS) : "memory"); }

template <int NR>
__global__ void __launch_bounds__(GT_THREADS, 1)
gemv_tc_kernel(const __grid_constant__ CUtensorMap map_w, const float* __restrict__ x, const float* __restrict__ bias,
               float* __restrict__ out, int R, int N, int K, int rows_box) {
  extern __shared__ uint8_t gt_raw[];
  const uint32_t raw_addr = smem_u32(gt_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;
  uint8_t* smem = gt_raw + (base - raw_addr);
  const uint32_t sB = base + GT_OFF_B;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + GT_OFF_BAR);
  const uint32_t bar0 = smem_u32(bars);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (GT_NSTAGE + s); };
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int s = 0; s < GT_NSTAGE; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 1);
    }
    fence_mbar_init();
    tma_prefetch_desc(&map_w);
  }
  for (int i = tid; i < GT_B_BYTES / 16; i += GT_THREADS) *reinterpret_cast<uint4*>(smem + GT_OFF_B + i * 16) = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();

  // row slice of this CTA, in groups of 64 weight rows (one 64 x 8 accumulator per group)
  const int per = (N + gridDim.x - 1) / gridDim.x;
  int lo = blockIdx.x * per, hi = min(N, lo + per);
  if (lo > hi) lo = hi;
  const int n_groups = (hi - lo + 63) / 64;
  const int kblocks = K / 64;
  int kbu = GT_STAGE / (rows_box * 128);  // k-blocks per ring unit
  if (kbu > kblocks) kbu = kblocks;
  const int units_per_group = (kblocks + kbu - 1) / kbu;

  if (tid == GT_CONS) {
    // ------------------------------------------------------------ producer: 2-D TMA boxes (64 k x rows_box weight rows)
    unsigned unit = 0;
    for (int g = 0; g < n_groups; ++g) {
      const int row0 = lo + g * 64;
      for (int u = 0; u < units_per_group; ++u, ++unit) {
        const int kb0 = u * kbu, nkb = min(kbu, kblocks - kb0);
        const int st = unit % GT_NSTAGE;
        mbar_wait(empty_bar(st), ((unit / GT_NSTAGE) & 1u) ^ 1u);
        mbar_arrive_expect_tx(full_bar(st), static_cast<uint32_t>(nkb * rows_box * 128));
        for (int i = 0; i < nkb; ++i)
          tma_load_2d(base + st * GT_STAGE + i * rows_box * 128, &map_w, full_bar(st), (kb0 + i) * 64, row0);
      }
    }
  } else if (tid < GT_CONS) {
    // ------------------------------------------------------------ consumer warpgroup
    // B operand: x -> fp16, [k-block][8 rows][128 B] with the 16-byte chunks XOR-swizzled by the row (rows >= R stay zero)
    for (int v = tid; v < K / 8; v += GT_CONS) {
      const int kb = v >> 3, c = v & 7;
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        if (r < R) {
          const float4 a0 = __ldcg(reinterpret_cast<const float4*>(x + static_cast<long long>(r) * K + v * 8));
          const float4 a1 = __ldcg(reinterpret_cast<const float4*>(x + static_cast<long long>(r) * K + v * 8 + 4));
          __half2 h0 = __floats2half2_rn(a0.x, a0.y), h1 = __floats2half2_rn(a0.z, a0.w);
          __half2 h2 = __floats2half2_rn(a1.x, a1.y), h3 = __floats2half2_rn(a1.z, a1.w);
          uint4 u4;
          u4.x = *reinterpret_cast<uint32_t*>(&h0); u4.y = *reinterpret_cast<uint32_t*>(&h1);
          u4.z = *reinterpret_cast<uint32_t*>(&h2); u4.w = *reinterpret_cast<uint32_t*>(&h3);
          *reinterpret_cast<uint4*>(smem + GT_OFF_B + kb * 1024 + r * 128 + ((c ^ r) << 4)) = u4;
        }
      }
    }
    fence_proxy_async_smem();
    gt_cons_sync();
    unsigned unit = 0;
    for (int g = 0; g < n_groups; ++g) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int u = 0; u < units_per_group; ++u, ++unit) {
        const int kb0 = u * kbu, nkb = min(kbu, kblocks - kb0);
        const int st = unit % GT_NSTAGE;
        mbar_wait(full_bar(st), (unit / GT_NSTAGE) & 1u);
        wgmma_fence();
        for (int i = 0; i < nkb; ++i) {
          const uint64_t da = make_desc_sw128(base + st * GT_STAGE + i * rows_box * 128, 1024);
          const uint64_t db = make_desc_sw128(sB + (kb0 + i) * 1024, 1024);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_ss<8, 0, 0>(acc, da + 2u * k, db + 2u * k, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (tid == 0) mbar_arrive(empty_bar(st));
      }
      wgmma_reg_fence(acc);
      // acc[0..1]: weight row 16 warp + lane / 4, x rows 2 (lane % 4) + {0,1}; acc[2..3]: weight row + 8
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = lo + g * 64 + warp * 16 + (lane >> 2) + 8 * h;
        if (n < hi) {
          const float b = bias != nullptr ? __ldg(bias + n) : 0.f;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int r = 2 * (lane & 3) + e;
            if (r < R && r < NR) out[static_cast<long long>(r) * N + n] = acc[2 * h + e] + b;
          }
        }
      }
    }
  }
}

}  // namespace

// x fp32 [R, K] (device), w fp16 [N, K] (device), out fp32 [R, N] (device).  Returns the average kernel time in microseconds.
float gemv_tc_debug_run(const float* x, const __half* w, const float* bias, float* out, int R, int N, int K, int num_sms,
                        int iters, cudaStream_t stream) {
  WISB_REQUIRE(R >= 1 && R <= 8 && K % 64 == 0 && K <= 5120 && N >= 1, "gemv_tc: 1..8 rows, K multiple of 64 and <= 5120");
  const int per = (N + num_sms - 1) / num_sms;
  int rows_box = round_up(per < 64 ? per : 64, 8);
  static std::atomic<unsigned long long> once{0};
  once_per_device(once, [] {
    WISB_CUDA(cudaFuncSetAttribute(gemv_tc_kernel<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, GT_SMEM));
    WISB_CUDA(cudaFuncSetAttribute(gemv_tc_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, GT_SMEM));
  });
  CUtensorMap map;
  make_tmap_f16_2d(&map, w, K, N, K, 64, rows_box);
  cudaEvent_t e0, e1;
  WISB_CUDA(cudaEventCreate(&e0));
  WISB_CUDA(cudaEventCreate(&e1));
  auto launch = [&] {
    if (R <= 5)
      gemv_tc_kernel<5><<<num_sms, GT_THREADS, GT_SMEM, stream>>>(map, x, bias, out, R, N, K, rows_box);
    else
      gemv_tc_kernel<8><<<num_sms, GT_THREADS, GT_SMEM, stream>>>(map, x, bias, out, R, N, K, rows_box);
  };
  launch();
  WISB_CUDA(cudaGetLastError());
  WISB_CUDA(cudaEventRecord(e0, stream));
  for (int i = 0; i < iters; ++i) launch();
  WISB_CUDA(cudaEventRecord(e1, stream));
  WISB_CUDA(cudaStreamSynchronize(stream));
  float ms = 0.f;
  WISB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return iters > 0 ? ms * 1e3f / iters : 0.f;
}

}  // namespace wisb
