// Batched log-mel front end for sm_90a.
//
// Replaces wis/audio.py:28-51 (pad_or_trim) and :72-103 (log_mel_spectrogram):
//   hann(400) periodic, STFT n_fft=400 hop=160 center/reflect, |.|^2 of the first 3000 frames, NMx201 Slaney mel
//   filterbank (NM = 80, or 128 for the large-v3 family), log10(clamp 1e-10), max(x, utterance_max - 8), (x + 4) / 4.
// Differences in HOW (not what): zero-padding / trimming to 480000 samples and the optional s16 -> f32 conversion are
// fused into the frame gather (the padded PCM is never materialised); the 400-point real DFT is evaluated directly
// using the even/odd symmetry of the windowed frame (201 x 200 MACs per frame instead of an FFT -- single-pass TF32
// tensor cores miss the 1e-4 parity bar, see BASELINE.md section 2), from fp32 samples and fp32 twiddle tables into
// fp64 accumulators (an fp32 chain is up to 4e-4 off float64 in the quiet bins beside a loud tone); frames that lie
// wholly in the zero padding skip the DFT.  HBM traffic per window: <= 1.92 MB PCM in, 0.96 MB out at 80 bins / 1.54 MB at 128 (+ the same again
// re-read/written by the clamp pass).
#include <math.h>

#include <vector>

#include "kernels.h"
#include "mel_filters_table.inc"
#include "mel_filters_table128.inc"

namespace wisb {

namespace {

constexpr int N_FFT = 400;
constexpr int HOP = 160;
constexpr int N_BINS = 201;
constexpr int BINS_PAD = 208;  // 4 x 52
constexpr int FT = 32;         // frames per CTA
constexpr int SPAN = (FT - 1) * HOP + N_FFT;  // 5360 samples feed one CTA
constexpr int KQ = 52;
constexpr int LM_THREADS = 224;  // 208 workers (52 bin-quads x 4 frame groups) + 16 helpers
constexpr int P_LD = BINS_PAD + 1;

// each bin count has its own tables, so front ends of both kinds can run in one process
__constant__ int c_mel_start[80];
__constant__ int c_mel_len[80];
__constant__ float c_mel_w[80][MEL_MAXNZ];
__constant__ int c_mel128_start[128];
__constant__ int c_mel128_len[128];
__constant__ float c_mel128_w[128][MEL_MAXNZ];

template <int NM>
struct MelTables;
template <>
struct MelTables<80> {
  static __device__ __forceinline__ int start(int m) { return c_mel_start[m]; }
  static __device__ __forceinline__ int len(int m) { return c_mel_len[m]; }
  static __device__ __forceinline__ float w(int m, int q) { return c_mel_w[m][q]; }
};
template <>
struct MelTables<128> {
  static __device__ __forceinline__ int start(int m) { return c_mel128_start[m]; }
  static __device__ __forceinline__ int len(int m) { return c_mel128_len[m]; }
  static __device__ __forceinline__ float w(int m, int q) { return c_mel128_w[m][q]; }
};

__device__ __forceinline__ unsigned f2ord(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

template <bool S16>
__device__ __forceinline__ float load_sample(const void* pcm, long long off, int n_eff, long long idx) {
  // idx indexes the (virtual) 480000-sample padded window with torch.stft's reflect padding around it
  if (idx < 0) idx = -idx;
  if (idx >= N_SAMPLES) idx = 2LL * (N_SAMPLES - 1) - idx;
  if (idx >= n_eff) return 0.f;
  if (S16) return static_cast<float>(reinterpret_cast<const short*>(pcm)[off + idx]) * (1.0f / 32768.0f);
  return reinterpret_cast<const float*>(pcm)[off + idx];
}

// twiddle tables: tw[n][k] = hann[n] * cos(2 pi k n / 400), ts[n][k] = hann[n] * sin(2 pi k n / 400), n in [0,200]
template <int NM, bool S16>
__global__ void __launch_bounds__(LM_THREADS)
logmel_power_kernel(const void* __restrict__ pcm, const long long* __restrict__ offsets, const int* __restrict__ n_samples,
                    const float* __restrict__ tw, const float* __restrict__ ts, float* __restrict__ mel,
                    unsigned* __restrict__ gmax) {
  __shared__ float xs[SPAN];
  __shared__ float pw[FT][P_LD];
  __shared__ float red[LM_THREADS / 32];
  const int b = blockIdx.y;
  const int f0 = blockIdx.x * FT;
  const int tid = threadIdx.x;
  const int n_eff = min(n_samples[b], N_SAMPLES);
  const long long off = offsets[b];
  const long long s0 = static_cast<long long>(f0) * HOP - N_FFT / 2;  // first padded-window index this CTA touches
  float* out = mel + static_cast<long long>(b) * NM * N_FRAMES;

  // frames wholly inside the zero padding: power == 0 -> log10(clamp) == -10 exactly
  const bool all_zero = (s0 >= n_eff) && (s0 + SPAN <= N_SAMPLES);
  float local_max = -10.0f;
  if (all_zero) {
    for (int i = tid; i < NM * FT; i += LM_THREADS) {
      const int m = i / FT, f = f0 + (i % FT);
      if (f < N_FRAMES) out[m * N_FRAMES + f] = -10.0f;
    }
  } else {
    for (int i = tid; i < SPAN; i += LM_THREADS) xs[i] = load_sample<S16>(pcm, off, n_eff, s0 + i);
    __syncthreads();
    if (tid < KQ * 4) {
      const int kq = tid % KQ;
      const int fg = tid / KQ;  // 8 frames each
      // float64 accumulators: each product of two floats is exact in float64, so the only roundings left are the
      // fold's and the tables' (one each per term) -- a float32 chain loses the small bins next to a loud tone
      double re[4][8], im[4][8];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int f = 0; f < 8; ++f) re[j][f] = im[j][f] = 0.0;
      const float* xb = xs + fg * 8 * HOP;
#pragma unroll 2
      for (int n = 0; n <= N_FFT / 2; ++n) {
        double c[4], s[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          c[j] = __ldg(tw + n * BINS_PAD + kq + KQ * j);
          s[j] = __ldg(ts + n * BINS_PAD + kq + KQ * j);
        }
#pragma unroll
        for (int f = 0; f < 8; ++f) {
          const float a = xb[f * HOP + n];
          const float bq = (n == 0 || n == N_FFT / 2) ? 0.f : xb[f * HOP + N_FFT - n];
          const double ev = a + bq, od = a - bq;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            re[j][f] = fma(ev, c[j], re[j][f]);
            im[j][f] = fma(od, s[j], im[j][f]);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int f = 0; f < 8; ++f)
          pw[fg * 8 + f][kq + KQ * j] = static_cast<float>(re[j][f] * re[j][f] + im[j][f] * im[j][f]);
    }
    __syncthreads();
    for (int i = tid; i < NM * FT; i += LM_THREADS) {
      const int m = i / FT, fl = i % FT;
      const int f = f0 + fl;
      const int st = MelTables<NM>::start(m), ln = MelTables<NM>::len(m);
      float acc = 0.f;
      for (int q = 0; q < ln; ++q) acc = fmaf(MelTables<NM>::w(m, q), pw[fl][st + q], acc);
      const float lg = log10f(fmaxf(acc, 1e-10f));
      if (f < N_FRAMES) {
        out[m * N_FRAMES + f] = lg;
        local_max = fmaxf(local_max, lg);
      }
    }
  }
  local_max = warp_max(local_max);
  if ((tid & 31) == 0) red[tid >> 5] = local_max;
  __syncthreads();
  if (tid == 0) {
    float m = red[0];
    for (int w = 1; w < LM_THREADS / 32; ++w) m = fmaxf(m, red[w]);
    atomicMax(gmax + b, f2ord(m));
  }
}

__global__ void logmel_finalize_kernel(float* __restrict__ mel, const unsigned* __restrict__ gmax, int per_utt4) {
  const int b = blockIdx.y;
  const float floor_v = ord2f(gmax[b]) - 8.0f;
  float4* p = reinterpret_cast<float4*>(mel) + static_cast<long long>(b) * per_utt4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < per_utt4; i += gridDim.x * blockDim.x) {
    float4 v = p[i];
    v.x = (fmaxf(v.x, floor_v) + 4.0f) * 0.25f;
    v.y = (fmaxf(v.y, floor_v) + 4.0f) * 0.25f;
    v.z = (fmaxf(v.z, floor_v) + 4.0f) * 0.25f;
    v.w = (fmaxf(v.w, floor_v) + 4.0f) * 0.25f;
    p[i] = v;
  }
}

}  // namespace

size_t logmel_table_floats() { return 2ull * (N_FFT / 2 + 1) * BINS_PAD; }

// tables_dev: [2][201][208] f32 (hann-weighted cos / sin); uploads the n_mels-bin filterbank to __constant__ memory too
void logmel_init_tables(float* tables_dev, int n_mels, cudaStream_t stream) {
  WISB_REQUIRE(n_mels == 80 || n_mels == 128, "log-mel: n_mels must be 80 or 128");
  const int rows = N_FFT / 2 + 1;
  std::vector<float> h(2ull * rows * BINS_PAD, 0.f);
  for (int n = 0; n < rows; ++n) {
    const double w = 0.5 - 0.5 * cos(2.0 * M_PI * n / N_FFT);  // periodic Hann, wis/audio.py:93
    const float wf = static_cast<float>(w);
    for (int k = 0; k < N_BINS; ++k) {
      const int r = (k * n) % N_FFT;  // exact argument reduction
      h[(0ull * rows + n) * BINS_PAD + k] = static_cast<float>(static_cast<double>(wf) * cos(2.0 * M_PI * r / N_FFT));
      h[(1ull * rows + n) * BINS_PAD + k] = static_cast<float>(static_cast<double>(wf) * sin(2.0 * M_PI * r / N_FFT));
    }
  }
  WISB_CUDA(cudaMemcpyAsync(tables_dev, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
  if (n_mels == 80) {
    WISB_CUDA(cudaMemcpyToSymbolAsync(c_mel_start, kMelStart, sizeof(kMelStart), 0, cudaMemcpyHostToDevice, stream));
    WISB_CUDA(cudaMemcpyToSymbolAsync(c_mel_len, kMelLen, sizeof(kMelLen), 0, cudaMemcpyHostToDevice, stream));
    WISB_CUDA(cudaMemcpyToSymbolAsync(c_mel_w, kMelW, sizeof(kMelW), 0, cudaMemcpyHostToDevice, stream));
  } else {
    WISB_CUDA(cudaMemcpyToSymbolAsync(c_mel128_start, kMel128Start, sizeof(kMel128Start), 0, cudaMemcpyHostToDevice, stream));
    WISB_CUDA(cudaMemcpyToSymbolAsync(c_mel128_len, kMel128Len, sizeof(kMel128Len), 0, cudaMemcpyHostToDevice, stream));
    WISB_CUDA(cudaMemcpyToSymbolAsync(c_mel128_w, kMel128W, sizeof(kMel128W), 0, cudaMemcpyHostToDevice, stream));
  }
  WISB_CUDA(cudaStreamSynchronize(stream));  // h goes out of scope
}

void logmel_run(const void* pcm, int pcm_is_s16, const long long* offsets_dev, const int* n_samples_dev, int B,
                int n_mels, const float* tables_dev, float* mel, unsigned* max_ws, cudaStream_t stream) {
  WISB_REQUIRE(n_mels == 80 || n_mels == 128, "log-mel: n_mels must be 80 or 128");
  const int rows = N_FFT / 2 + 1;
  WISB_CUDA(cudaMemsetAsync(max_ws, 0, sizeof(unsigned) * B, stream));
  dim3 grid(cdiv(N_FRAMES, FT), B);
  const float* tw = tables_dev;
  const float* ts = tables_dev + static_cast<size_t>(rows) * BINS_PAD;
  auto kernel = n_mels == 80 ? (pcm_is_s16 ? logmel_power_kernel<80, true> : logmel_power_kernel<80, false>)
                             : (pcm_is_s16 ? logmel_power_kernel<128, true> : logmel_power_kernel<128, false>);
  kernel<<<grid, LM_THREADS, 0, stream>>>(pcm, offsets_dev, n_samples_dev, tw, ts, mel, max_ws);
  WISB_CUDA(cudaGetLastError());
  const int per_utt4 = n_mels * N_FRAMES / 4;
  dim3 g2(cdiv(per_utt4, 256 * 4), B);
  logmel_finalize_kernel<<<g2, 256, 0, stream>>>(mel, max_ws, per_utt4);
  WISB_CUDA(cudaGetLastError());
}

}  // namespace wisb
