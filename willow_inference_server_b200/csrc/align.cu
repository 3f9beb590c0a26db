// Whisper.align post-processing on the device: the standardise / median-filter / head-mean of the captured alignment-head
// attention, dynamic time warping with an on-device backtrace, and the text-token probabilities.  The rules are
// transformers' (models/whisper/generation_whisper.py: _extract_token_timestamps, _median_filter,
// _dynamic_time_warping); DESIGN.md section 5 records the pinning.
#include "decoder.cuh"

namespace wisb {

namespace {

constexpr int AF_THREADS = 128;
constexpr int DTW_THREADS = 512;  // >= n_text_ctx + 1 rows of the cost matrix
constexpr int DTW_MAX_SMEM = 227 * 1024;

// in place: x[r][f] = (x[r][f] - mean_r) / std_r per (utterance, head, frame), two passes in row order, population std
__global__ void __launch_bounds__(AF_THREADS)
align_std_kernel(float* __restrict__ cap, const int* __restrict__ n_text, const int* __restrict__ n_frames, int A, int n_max,
                 int f_max) {
  const int u = blockIdx.z, a = blockIdx.y;
  const int f = blockIdx.x * AF_THREADS + threadIdx.x;
  const int n = n_text[u];
  if (n <= 0 || f >= n_frames[u]) return;
  const int R = n + 1;
  float* x = cap + (static_cast<long long>(u) * A + a) * (n_max + 1) * f_max + f;
  float s = 0.f;
  for (int r = 0; r < R; ++r) s += x[static_cast<long long>(r) * f_max];
  const float mean = s / R;
  float q = 0.f;
  for (int r = 0; r < R; ++r) {
    const float c = x[static_cast<long long>(r) * f_max] - mean;
    q += c * c;
  }
  const float sd = sqrtf(q / R);
  for (int r = 0; r < R; ++r) x[static_cast<long long>(r) * f_max] = (x[static_cast<long long>(r) * f_max] - mean) / sd;
}

// mat[u][r][f] = mean over heads (head order) of the median of the width-W reflect-padded window around f; the window is
// sorted in registers by an odd-even transposition network (the median of a sort is exact whatever the network)
template <int W>
__global__ void __launch_bounds__(AF_THREADS)
align_median_kernel(const float* __restrict__ cap, float* __restrict__ mat, const int* __restrict__ n_text,
                    const int* __restrict__ n_frames, int A, int n_max, int f_max) {
  const int u = blockIdx.z, r = blockIdx.y;
  const int f = blockIdx.x * AF_THREADS + threadIdx.x;
  const int n = n_text[u], F = n_frames[u];
  if (n <= 0 || r > n || f >= F) return;
  constexpr int P = W / 2;
  const bool identity = F <= P;
  float acc = 0.f;
  for (int a = 0; a < A; ++a) {
    const float* x = cap + ((static_cast<long long>(u) * A + a) * (n_max + 1) + r) * f_max;
    float med;
    if (identity) {
      med = x[f];
    } else {
      float v[W];
#pragma unroll
      for (int k = 0; k < W; ++k) {
        int j = f - P + k;
        j = j < 0 ? -j : j;
        j = j >= F ? 2 * (F - 1) - j : j;
        v[k] = x[j];
      }
#pragma unroll
      for (int pass = 0; pass < W; ++pass)
#pragma unroll
        for (int k = pass & 1; k + 1 < W; k += 2) {
          const float lo = fminf(v[k], v[k + 1]), hi = fmaxf(v[k], v[k + 1]);
          v[k] = lo;
          v[k + 1] = hi;
        }
      med = v[P];
    }
    acc += med;
  }
  mat[(static_cast<long long>(u) * (n_max + 1) + r) * f_max + f] = acc / A;
}

// one CTA per utterance: cost = fp32 DTW on -mat over anti-diagonals k = i + j (thread i owns row i; the last three
// diagonals live in shared memory), 2-bit trace packed in shared memory, serial backtrace by thread 0.  Every cell reads
// only its three finished predecessors, so the costs, the traces and the path equal the serial column loop's.
__global__ void __launch_bounds__(DTW_THREADS)
align_dtw_kernel(const float* __restrict__ mat, const int* __restrict__ n_text, const int* __restrict__ n_frames, int n_max,
                 int f_max, int* __restrict__ path, int path_stride, int* __restrict__ path_len) {
  extern __shared__ uint32_t dtw_smem[];
  const int u = blockIdx.x, i = threadIdx.x;
  const int n = n_text[u];
  if (n <= 0) {
    if (i == 0) path_len[u] = 0;
    return;
  }
  const int R = n + 1, F = n_frames[u];
  const int words = (R * F + 15) / 16;
  uint32_t* trace = dtw_smem;
  float* diag = reinterpret_cast<float*>(dtw_smem + words);  // [3][R + 1]: diagonal k in slot k % 3
  for (int w = i; w < words; w += DTW_THREADS) trace[w] = 0u;
  const float* m = mat + static_cast<long long>(u) * (n_max + 1) * f_max;
  for (int k = 0; k <= R + F; ++k) {
    __syncthreads();
    if (i <= R) {
      const int j = k - i;
      float c;
      if (i == 0) {
        c = k == 0 ? 0.f : INFINITY;
      } else if (j <= 0 || j > F) {
        c = INFINITY;
      } else {
        const float* d1 = diag + ((k + 2) % 3) * (R + 1);  // diagonal k - 1
        const float* d2 = diag + ((k + 1) % 3) * (R + 1);  // diagonal k - 2
        const float c0 = d2[i - 1], c1 = d1[i - 1], c2 = d1[i];
        float best;
        uint32_t t;
        if (c0 < c1 && c0 < c2) {
          best = c0;
          t = 0;
        } else if (c1 < c0 && c1 < c2) {
          best = c1;
          t = 1;
        } else {
          best = c2;
          t = 2;
        }
        c = -m[static_cast<long long>(i - 1) * f_max + (j - 1)] + best;
        const int cell = (i - 1) * F + (j - 1);
        if (t) atomicOr(&trace[cell >> 4], t << (2 * (cell & 15)));
      }
      diag[(k % 3) * (R + 1) + i] = c;
    }
  }
  __syncthreads();
  if (i != 0) return;
  // backtrace with trace[0, :] = 2 and trace[:, 0] = 1
  auto step = [&](int& ii, int& jj) {
    int t;
    if (ii == 0) t = 2;
    else if (jj == 0) t = 1;
    else {
      const int cell = (ii - 1) * F + (jj - 1);
      t = (trace[cell >> 4] >> (2 * (cell & 15))) & 3;
    }
    if (t == 0) { --ii; --jj; }
    else if (t == 1) --ii;
    else --jj;
  };
  int len = 0;
  for (int ii = R, jj = F; ii > 0 || jj > 0; step(ii, jj)) ++len;
  if (len > path_stride) len = path_stride;  // (the host requires path_stride >= R + F, the longest possible path)
  int* out = path + static_cast<long long>(u) * path_stride * 2;
  int idx = len - 1;
  for (int ii = R, jj = F; (ii > 0 || jj > 0) && idx >= 0; step(ii, jj), --idx) {
    out[2 * idx] = ii - 1;
    out[2 * idx + 1] = jj - 1;
  }
  path_len[u] = len;
}

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
  v = is_max ? warp_max(v) : warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = is_max ? -INFINITY : 0.f;
  for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
  return r;
}

__global__ void __launch_bounds__(256)
align_token_probs_kernel(const float* __restrict__ logits, long long ldl, const int* __restrict__ row_pos,
                         const int* __restrict__ text, int text_stride, const int* __restrict__ n_text, int rows_per_utt,
                         int s0, int eot, float* __restrict__ probs) {
  __shared__ float red[8];
  const int row = blockIdx.x, u = row / rows_per_utt;
  const int i = row_pos[row] - s0;
  if (i < 0 || i >= n_text[u]) return;
  const float* lg = logits + static_cast<long long>(row) * ldl;
  float m = -INFINITY;
  for (int v = threadIdx.x; v < eot; v += blockDim.x) m = fmaxf(m, lg[v]);
  m = block_reduce(m, true, red);
  float s = 0.f;
  for (int v = threadIdx.x; v < eot; v += blockDim.x) s += expf(lg[v] - m);
  s = block_reduce(s, false, red);
  if (threadIdx.x == 0) probs[static_cast<long long>(u) * text_stride + i] = expf(lg[text[u * text_stride + i]] - m) / s;
}

template <int W>
void median_launch(const float* cap, float* mat, const int* n_text, const int* n_frames, int n_utt, int A, int n_max, int f_max,
                   cudaStream_t s) {
  align_median_kernel<W><<<dim3(cdiv(f_max, AF_THREADS), n_max + 1, n_utt), AF_THREADS, 0, s>>>(cap, mat, n_text, n_frames, A,
                                                                                              n_max, f_max);
}

}  // namespace

int align_dtw_smem(int rows, int frames) { return ((rows * frames + 15) / 16) * 4 + 3 * (rows + 1) * 4; }

void align_filter_run(float* cap, float* mat, const int* n_text, const int* n_frames, int n_utt, int A, int n_max, int f_max,
                      int width, cudaStream_t s) {
  WISB_REQUIRE(width >= 1 && width <= 31 && width % 2 == 1, "median_filter_width must be odd and in [1, 31]");
  align_std_kernel<<<dim3(cdiv(f_max, AF_THREADS), A, n_utt), AF_THREADS, 0, s>>>(cap, n_text, n_frames, A, n_max, f_max);
  WISB_CUDA(cudaGetLastError());
  switch (width) {
    case 1: median_launch<1>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 3: median_launch<3>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 5: median_launch<5>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 7: median_launch<7>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 9: median_launch<9>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 11: median_launch<11>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 13: median_launch<13>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 15: median_launch<15>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 17: median_launch<17>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 19: median_launch<19>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 21: median_launch<21>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 23: median_launch<23>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 25: median_launch<25>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 27: median_launch<27>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    case 29: median_launch<29>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
    default: median_launch<31>(cap, mat, n_text, n_frames, n_utt, A, n_max, f_max, s); break;
  }
  WISB_CUDA(cudaGetLastError());
}

void align_dtw_run(const float* mat, const int* n_text, const int* n_frames, int n_utt, int n_max, int f_max, int* path,
                   int path_stride, int* path_len, cudaStream_t s) {
  WISB_REQUIRE(n_max + 1 <= DTW_THREADS - 1, "alignment: more than 510 text rows");
  const int smem = align_dtw_smem(n_max + 1, f_max);
  WISB_REQUIRE(smem <= DTW_MAX_SMEM, "alignment: DTW trace does not fit in shared memory");
  static std::atomic<unsigned long long> once{0};
  once_per_device(once, [] {
    WISB_CUDA(cudaFuncSetAttribute(align_dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DTW_MAX_SMEM));
  });
  align_dtw_kernel<<<n_utt, DTW_THREADS, smem, s>>>(mat, n_text, n_frames, n_max, f_max, path, path_stride, path_len);
  WISB_CUDA(cudaGetLastError());
}

void align_token_probs_run(const float* logits, long long ldl, const int* row_pos, const int* text, int text_stride,
                           const int* n_text, int n_utt, int rows_per_utt, int s0, int eot, float* probs, cudaStream_t s) {
  align_token_probs_kernel<<<n_utt * rows_per_utt, 256, 0, s>>>(logits, ldl, row_pos, text, text_stride, n_text, rows_per_utt,
                                                               s0, eot, probs);
  WISB_CUDA(cudaGetLastError());
}

}  // namespace wisb
