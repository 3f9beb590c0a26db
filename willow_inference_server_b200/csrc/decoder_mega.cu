// Persistent decoder-pass kernel ("megakernel"): one cooperative launch runs a whole decoder forward pass
// (embedding, L x {LN+QKV, self-attention, out-proj, LN+cross-Q, cross-attention, out-proj, LN+fc1+GELU, fc2},
// final LN + vocabulary projection) for <= 8 rows, instead of ~260 dependent kernel launches.
//
// Why: at <= 8 rows the pass is bound by streaming 1.8 GB of fp16 decoder weights (SURVEY.md section 8d), but a chain
// of per-op kernels exposes launch + HBM latency ~260 times per pass, even with PDL.  Here
//   * one CTA per SM, every CTA owns a fixed column slice of every weight matrix;
//   * a dedicated producer thread per CTA walks the (static) list of weight chunks of ALL phases and streams them into a
//     2-stage shared-memory ring with cp.async.bulk (TMA, L2 evict-first) + mbarrier complete_tx -- it never waits for
//     activations, so the HBM stream keeps running across phase boundaries.  (Two stages on purpose: with 5 stages the
//     180 KB of bulk copies in flight per SM queued every demand load -- activation reloads, K/V rows -- behind them.)
//   * consumer warps wait only on (a) the ring and (b) a flag-based grid barrier between phases (per-CTA epoch flags,
//     no atomics), and read activations with L1-bypassing loads;
//   * activations stay fp32; LayerNorm (single-pass sum / sum-of-squares statistics in fp32) is applied in registers while staging x.
// Mapping inside a GEMV phase: thread = one 16-byte K-slice (8 elements) of the CTA's columns; it keeps x[r][8] of all
// rows in registers and streams the CTA's <= 12 columns through them (weights from the ring), then a transposing warp
// reduction + one shared-memory hop produce the outputs.
//
// Reference semantics: decoder step of ctranslate2.models.Whisper.generate (main.py:687-692);
// architecture [HF] modeling_whisper.py:417-508, :650-700, :966-971.
#include <cooperative_groups.h>

#include "decoder.cuh"
#include "ptx.cuh"

namespace wisb {

namespace {

constexpr int MG_CONS_WARPS = 7;                        // consumer warps
constexpr int MG_CONS = MG_CONS_WARPS * 32;             // 320 consumer threads
constexpr int MG_THREADS = MG_CONS + 32;                // + producer warp (lane 0 only)
constexpr int MG_KC_MAX = 1536;
constexpr int MG_STAGE_BYTES = 12 * MG_KC_MAX * 2;      // 36864: up to 12 weight-row chunks (or 288 keys of K / V)
constexpr int MG_NSTAGE = 2;
constexpr int MG_CA_KEYS_MAX = MG_STAGE_BYTES / 128;    // 288 keys per K (or V) chunk
constexpr int MG_SCRATCH = 29696;                       // self-attention V rows + probabilities / cross-attention merge
constexpr int MG_SLOT_BYTES = MG_CONS_WARPS * 448 * 2;  // per-warp cache-slot table of the warp's self-attention task
constexpr int MG_LY_STRIDE = 704;
constexpr int MG_LY_BYTES = 2 * MG_LY_STRIDE;           // double-buffered copy of the layer descriptor
constexpr int MG_RED_FLOATS = (2 * 2 + 1) * MG_CONS_WARPS * 32;  // 2 buffers x 2 sets + LN partials
constexpr int MG_SMEM = MG_NSTAGE * MG_STAGE_BYTES + 1024 + MG_RED_FLOATS * 4 + 4224 + MG_SCRATCH + MG_SLOT_BYTES + MG_LY_BYTES;
static_assert(MG_SMEM <= 232448, "decoder pass: shared memory");
static_assert(sizeof(MegaLayer) % 16 == 0 && sizeof(MegaLayer) <= MG_LY_STRIDE, "layer descriptor is copied with 16-byte cp.async");
// columns a thread accumulates per unit: the transposing reduction handles GP * NR <= 32 values
__host__ __device__ constexpr int mg_gp(int nr) { return 32 / nr < 6 ? 32 / nr : 6; }
// accumulator sets per thread: 2 x 6 columns for <= 5 rows (the stage holds 12 weight-row chunks), 1 x 4 for 8 rows
__host__ __device__ constexpr int mg_nset(int nr) { return nr <= 5 ? 2 : 1; }

__device__ __forceinline__ float ldcg_f(const float* p) { return __ldcg(p); }
__device__ __forceinline__ float4 ldcg_f4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ float2 ldcg_f2(const float* p) { return __ldcg(reinterpret_cast<const float2*>(p)); }

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void cons_sync() { asm volatile("bar.sync 1, %0;" ::"n"(MG_CONS) : "memory"); }

// in: lane l holds v[0..31]; out: v[0] of lane l = sum over all lanes of their v[l]
__device__ __forceinline__ float warp_transpose_reduce32(float (&v)[32], int lane) {
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

// Row geometry.  Normal step: every row is at position st->pos and owns cache slot r.  Prompt prefill (pf_len > 0): the
// pass carries the first pf_len prompt positions of each utterance as rows (utterance-major), all written into the cache
// slot of the utterance's first beam, so the whole prompt prefix costs ONE pass instead of pf_len passes.
__device__ __forceinline__ int row_pos(const MegaArgs& A, int r) { return A.pf_len > 0 ? r % A.pf_len : A.st->pos; }
__device__ __forceinline__ int row_slot(const MegaArgs& A, int r) { return A.pf_len > 0 ? (r / A.pf_len) * A.pf_slot_stride : r; }
__device__ __forceinline__ int row_token(const MegaArgs& A, int r) {
  return A.pf_len > 0 ? A.tokens[(r / A.pf_len) * A.pf_tok_stride + (r % A.pf_len)] : A.tokens[r];
}


// fp16 activation exchange of the warp-MMA pass: element (row r, feature k) of a [K/64 k-blocks][R rows][64] buffer stored in
// B-FRAGMENT order: inside a k-block, lane slot (g = r, t = (k / 2) % 4) holds the 8 words that lane of mma.m16n8k16 feeds
// to the 4 k-steps ({b0, b1} x 4), as two 16-byte planes -- exactly the B-operand image a consumer CTA wants in shared memory.
// Its reload is ONE bulk copy instead of a per-thread ld.global reload of the same bytes, and a lane fetches a whole k-block's fragments with two 16-byte loads.
__device__ __forceinline__ long long act16_off(int R, int r, int k) {
  // k-block: [plane p = k-steps {0,1} | {2,3}][lane slot r * 4 + t][4 words]: a warp's 16-byte fragment load touches 512
  // consecutive bytes (32-byte strides gave 2-way bank conflicts)
  const int kk = k & 63;
  const int w = (kk >> 4) * 2 + ((kk >> 3) & 1);  // word of the lane's 8: k-step * 2 + {b0, b1}
  return static_cast<long long>(k >> 6) * (R * 64) + (w >> 2) * (R * 32) + (r * 4 + ((kk >> 1) & 3)) * 8 + (w & 3) * 2 + (kk & 1);
}
// attention output of row r, features [col, col + 2): fp32 [R, d] (SIMT pass) or the fp16 exchange image (warp-MMA pass)
__device__ __forceinline__ void store_ctx2(const MegaArgs& A, int r, int col, float v0, float v1) {
  if (A.ctx16 != nullptr) {
    *reinterpret_cast<__half2*>(A.ctx16 + act16_off(A.R, r, col)) = __floats2half2_rn(v0, v1);
  } else {
    *reinterpret_cast<float2*>(A.ctx + static_cast<long long>(r) * A.d + col) = make_float2(v0, v1);
  }
}

struct Ring {
  uint32_t full0, empty0, data0;  // shared-memory addresses
  uint8_t* data;
  unsigned unit;                  // running unit counter (same sequence in producer and consumers)
  __device__ __forceinline__ uint32_t full(int s) const { return full0 + 8u * s; }
  __device__ __forceinline__ uint32_t empty(int s) const { return empty0 + 8u * s; }
};

// column slice of a GEMV phase owned by this CTA
__device__ __forceinline__ void cta_cols(int N, int& lo, int& hi) {
  const int per = (N + gridDim.x - 1) / gridDim.x;
  lo = blockIdx.x * per;
  hi = min(N, lo + per);
  if (lo > hi) lo = hi;
}
__device__ __forceinline__ void k_split(int K, int& n_chunks, int& kc) {
  n_chunks = (K + MG_KC_MAX - 1) / MG_KC_MAX;
  while (K % (8 * n_chunks) != 0) ++n_chunks;
  kc = K / n_chunks;
}
// thread parts: `wpp` warps cover the kc/8 K-slices once; with <= 5 warps per part two parts split the columns
__device__ __forceinline__ void part_geom(int kc, int& wpp, int& n_parts) {
  wpp = (kc / 8 + 31) / 32;
  n_parts = (2 * wpp <= MG_CONS_WARPS) ? 2 : 1;
}

// ------------------------------------------------------------------ producer side
__device__ __noinline__ void produce_gemv(Ring& rg, const MegaGemv& g, int gp) {
  int lo, hi, n_chunks, kc, wpp, n_parts;
  cta_cols(g.N, lo, hi);
  k_split(g.K, n_chunks, kc);
  part_geom(kc, wpp, n_parts);
  const int G = gp * n_parts;
  const uint64_t pol = l2_policy_evict_first();  // weights are read once per pass: do not let them flush the L2
  for (int g0 = lo; g0 < hi; g0 += G) {
    const int nc = min(G, hi - g0);
    for (int ch = 0; ch < n_chunks; ++ch) {
      const int st = rg.unit % MG_NSTAGE;
      mbar_wait(rg.empty(st), ((rg.unit / MG_NSTAGE) & 1u) ^ 1u);
      // one TMA request per unit: rows g0..g0+nc of a K-chunk are contiguous (multi-chunk matrices are stored
      // chunk-major [chunk][N][kc] by the engine at load time): many small copies (one per 2.5 KB row) would be bound by
      // the per-request rate of the copy engine.
      mbar_arrive_expect_tx(rg.full(st), static_cast<uint32_t>(nc * kc * 2));
      bulk_load_1d_hint(rg.data0 + st * MG_STAGE_BYTES, g.w + (static_cast<long long>(ch) * g.N + g0) * kc,
                        static_cast<uint32_t>(nc * kc * 2), rg.full(st), pol);
      ++rg.unit;
    }
  }
}

// cross-attention: task = (utterance, head, key split): the 1500 keys of a head are split over S CTAs (one K unit and
// one V unit of <= 288 keys each through the ring); the last split to finish merges the partials (split-K fix-up).
// (Splitting the keys spreads the online-softmax walk over 1500 keys, which is compute-bound, over several CTAs.)
struct CrossGeom {
  int S, KS, n_tasks;
};
__device__ __forceinline__ CrossGeom cross_geom(int n_utt, int H) {
  CrossGeom c;
  int s = gridDim.x / (n_utt * H);
  const int smin = (T_ENC + MG_CA_KEYS_MAX - 1) / MG_CA_KEYS_MAX;  // 6
  if (s < smin) s = smin;
  if (s > 16) s = 16;
  c.S = s;
  c.KS = ((T_ENC + s - 1) / s + 31) & ~31;  // whole 32-key MMA blocks per split (7 splits: 224 keys = one block per warp)
  c.n_tasks = n_utt * H * s;
  return c;
}

template <int NS = MG_NSTAGE>
__device__ __forceinline__ void produce_cross_impl(Ring& rg, const MegaArgs& A, const MegaLayer& ly) {
  const CrossGeom cg = cross_geom(A.n_utt, A.H);
  const uint64_t pol = l2_policy_evict_first();
  for (int task = blockIdx.x; task < cg.n_tasks; task += gridDim.x) {
    const int split = task % cg.S, uh = task / cg.S;
    const int t0 = split * cg.KS;
    // buffer has 1536 rows; keys >= 1500 are skipped by the consumer.  Rounding KS up can leave the last splits without
    // any rows (132 CTAs over 12 heads: 11 splits of 160 keys): their stages complete on the arrival alone
    const int nk = max(0, min(cg.KS, T_ENC_PAD - t0));
    const long long off = (static_cast<long long>(uh) * T_ENC_PAD + t0) * HEAD_DIM;
    for (int kv = 0; kv < 2; ++kv) {
      const int st = rg.unit % NS;
      mbar_wait(rg.empty(st), ((rg.unit / NS) & 1u) ^ 1u);
      mbar_arrive_expect_tx(rg.full(st), static_cast<uint32_t>(nk * HEAD_DIM * 2));
      if (nk > 0)
        bulk_load_1d_hint(rg.data0 + st * MG_STAGE_BYTES, (kv == 0 ? ly.ck : ly.cv) + off,
                          static_cast<uint32_t>(nk * HEAD_DIM * 2), rg.full(st), pol);
      ++rg.unit;
    }
  }
}

__device__ __noinline__ void produce_cross(Ring& rg, const MegaArgs& A, const MegaLayer& ly) { produce_cross_impl<MG_NSTAGE>(rg, A, ly); }

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// fine-grained event trace of thread 0 of ONE CTA over one layer (debug): (event id, SM clock) pairs collected in shared
// memory -- a clock read and two shared stores per event, far cheaper than a globaltimer read plus global stores -- and
// copied to trace[1024..] when the kernel ends.  s_tr[0] = events so far, < 0 while the window is closed.
__device__ __forceinline__ void trace_ev(const MegaArgs& A, int ctid, int* s_tr, int id) {
  if (A.trace != nullptr && ctid == 0) {
    const int i = s_tr[0];
    if (i >= 0 && i < A.trace_cap) {
      s_tr[1 + 2 * i] = id;
      s_tr[2 + 2 * i] = static_cast<int>(clock());
      s_tr[0] = i + 1;
    }
  }
}
__device__ __forceinline__ void trace_open(const MegaArgs& A, int ctid, int* s_tr, int layer) {
  if (A.trace != nullptr && ctid == 0 && static_cast<int>(blockIdx.x) == A.trace_cta && layer == A.trace_layer) s_tr[0] = 0;
}
__device__ __forceinline__ void trace_dump(const MegaArgs& A, int ctid, const int* s_tr) {
  if (A.trace != nullptr && ctid == 0 && static_cast<int>(blockIdx.x) == A.trace_cta) {
    const int n = s_tr[0] < 0 ? 0 : s_tr[0];
    A.trace[1024] = static_cast<unsigned long long>(n);
    for (int i = 0; i < 2 * n; ++i) A.trace[1025 + i] = static_cast<unsigned long long>(static_cast<unsigned>(s_tr[1 + i]));
  }
}

__device__ __forceinline__ void st_release_gpu(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Flag barrier: bar.sync orders the CTA's writes before thread 0's release store (cumulativity); every CTA publishes its
// epoch in its own 128-byte line and thread i polls CTA i's line with acquire loads -- no atomics, no all-thread fences.
__device__ __forceinline__ void grid_barrier(const MegaArgs& A, unsigned& epoch, int ctid, unsigned epoch0) {
  if (A.trace != nullptr && ctid == 0) {
    const unsigned long long t = globaltimer_ns();
    if (blockIdx.x == 0) A.trace[2 * (epoch - epoch0) + 1] = t;
    if (epoch - epoch0 < 264u) A.trace[2048 + blockIdx.x * 264 + (epoch - epoch0)] = t;  // arrival of every CTA at every barrier
  }
  cons_sync();
  ++epoch;
  if (A.barrier_mode == 1) {
    // one release-add per CTA on a shared counter, thread 0 spins on it (barrier_mode 0: the flag barrier); the counter equals epoch * gridDim.x whenever all CTAs have passed barrier `epoch`
    if (ctid == 0) {
      unsigned* counter = A.epoch_base + 8;
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
      const unsigned target = epoch * gridDim.x;
      while (static_cast<int>(ld_acquire_gpu(counter) - target) < 0) {
      }
    }
  } else {
    if (ctid == 0) st_release_gpu(A.flags + blockIdx.x * 32, epoch);
    if (ctid < static_cast<int>(gridDim.x)) {
      const unsigned* f = A.flags + ctid * 32;
      while (static_cast<int>(ld_acquire_gpu(f) - epoch) < 0) {
      }
    }
  }
  cons_sync();
  if (A.trace != nullptr && blockIdx.x == 0 && ctid == 0) A.trace[2 * (epoch - epoch0)] = globaltimer_ns();
}

// ------------------------------------------------------------------ consumer: one GEMV phase
// Thread (part, kv) keeps the K-slice kv of every row in registers and streams the unit's columns
// cj = part + n_parts * m (m < NSET * GP) through it.  LayerNorm is folded (s2 / folded bias precomputed at load):
//     LN(x) . w + bias = rstd * (sum_k x_k g_k w_k - mean * s2[n]) + biasf[n]
// so the row statistics are only needed in the epilogue and their reduction rides along with the first group's.
template <int NR>
__device__ __noinline__ void consume_gemv(Ring& rg, const MegaArgs& A, const MegaGemv& g_mem, const MegaLayer* ly, int ctid,
                                          float* s_red, float* s_stat) {
  const MegaGemv g = g_mem;  // descriptor into registers once (it lives in global memory)
  const uint32_t ring_data0 = rg.data0, ring_full0 = rg.full0, ring_empty0 = rg.empty0;
  unsigned unit = rg.unit;
  constexpr int GP = mg_gp(NR);
  constexpr int NSET = mg_nset(NR);
  constexpr int NACC = GP * NSET;
  const int lane = ctid & 31, warp = ctid >> 5;
  const int R = A.R;
  int lo, hi, n_chunks, kc, wpp, n_parts;
  cta_cols(g.N, lo, hi);
  k_split(g.K, n_chunks, kc);
  part_geom(kc, wpp, n_parts);
  const int G = NACC * n_parts;
  const int n_kvec = kc / 8;
  const int part = warp / wpp;
  const int kv = (warp - part * wpp) * 32 + lane;
  const bool active = part < n_parts && kv < n_kvec;
  const bool ln = g.ln_s2 != nullptr;
  int* s_tr = reinterpret_cast<int*>(s_stat + 912);  // [912, 1056): event trace
  trace_ev(A, ctid, s_tr, 1);
  float* s_bias = s_stat + 16;         // [<=384] bias (LN: folded bias) of this CTA's columns
  float* s_s2 = s_stat + 400;          // [<=384] LN fold vector of this CTA's columns
  float* s_xown = s_stat + 784;        // [8][16] residual-stream columns owned by this CTA (kept across phases)
  float* s_lnred = s_red + 2 * NSET * MG_CONS_WARPS * 32;  // [warps][32] per-warp partial row sums (LN)
  const int ncols = hi - lo;
  const bool pre = ncols <= 384;  // the vocabulary projection has 351 columns per CTA
  if (pre) {
    for (int i = ctid; i < ncols; i += MG_CONS) {
      s_bias[i] = g.bias != nullptr ? __ldg(g.bias + lo + i) : 0.f;
      if (ln) s_s2[i] = __ldg(g.ln_s2 + lo + i);
    }
  }
  float acc[NACC][NR];
  float xv[NR][8], xn[NR][8];
  float sx[NR], sxx[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) sx[r] = sxx[r] = 0.f;
  auto load_x = [&](float (&dst)[NR][8], int ch) {
    const int k = ch * kc + kv * 8;
#pragma unroll
    for (int r = 0; r < NR; ++r) {
#pragma unroll
      for (int i = 0; i < 8; ++i) dst[r][i] = 0.f;
      if (active && r < R) {
        const float4 x0 = ldcg_f4(g.x + static_cast<long long>(r) * g.K + k), x1 = ldcg_f4(g.x + static_cast<long long>(r) * g.K + k + 4);
        dst[r][0] = x0.x; dst[r][1] = x0.y; dst[r][2] = x0.z; dst[r][3] = x0.w;
        dst[r][4] = x1.x; dst[r][5] = x1.y; dst[r][6] = x1.z; dst[r][7] = x1.w;
      }
    }
  };
  int grp_idx = 0;
  for (int g0 = lo; g0 < hi; g0 += G) {
    const int nc = min(G, hi - g0);
#pragma unroll
    for (int m = 0; m < NACC; ++m)
#pragma unroll
      for (int r = 0; r < NR; ++r) acc[m][r] = 0.f;
    for (int ch = 0; ch < n_chunks; ++ch) {
      // ---- x[r][8] of this thread's K-slice: loaded once per phase (single-chunk K) or per chunk with the next
      //      chunk's loads already in flight (multi-chunk K, never with LayerNorm)
      if (g0 == lo || n_chunks > 1) {
        if (n_chunks == 1 || ch == 0) {
          load_x(xv, ch);
        } else {
#pragma unroll
          for (int r = 0; r < NR; ++r)
#pragma unroll
            for (int i = 0; i < 8; ++i) xv[r][i] = xn[r][i];
        }
        if (n_chunks > 1) load_x(xn, (ch + 1) % n_chunks);
        if (ln && active) {
          const int k = ch * kc + kv * 8;
          const float4 g0v = __ldg(reinterpret_cast<const float4*>(g.ln_g + k)), g1v = __ldg(reinterpret_cast<const float4*>(g.ln_g + k + 4));
          const float gg[8] = {g0v.x, g0v.y, g0v.z, g0v.w, g1v.x, g1v.y, g1v.z, g1v.w};
#pragma unroll
          for (int r = 0; r < NR; ++r)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              if (part == 0) {
                sx[r] += xv[r][i];
                sxx[r] = fmaf(xv[r][i], xv[r][i], sxx[r]);
              }
              xv[r][i] *= gg[i];
            }
        }
      }
      // ---- weights of this unit from the ring
      trace_ev(A, ctid, s_tr, 2);
      const int st = unit % MG_NSTAGE;
      mbar_wait(ring_full0 + 8u * st, (unit / MG_NSTAGE) & 1u);
      trace_ev(A, ctid, s_tr, 3);
      if (active) {
        const uint32_t stage = ring_data0 + st * MG_STAGE_BYTES;  // shared-space address: ld.shared, not generic loads
        // two columns at a time, k-element outermost: 2 * NR independent FMA chains are interleaved so the 4-cycle FMA
        // latency is covered by a single warp per scheduler (row-outer order left 8-deep dependent chains: 4x slower)
#pragma unroll
        for (int m = 0; m < NACC; m += 2) {
          const int c0 = part + n_parts * m, c1 = part + n_parts * (m + 1);
          if (c0 < nc) {
            const bool two = c1 < nc;
            const uint4 ua = lds128(stage + c0 * kc * 2 + kv * 16);
            const uint4 ub = two ? lds128(stage + c1 * kc * 2 + kv * 16) : make_uint4(0u, 0u, 0u, 0u);
            const __half2* ha = reinterpret_cast<const __half2*>(&ua);
            const __half2* hb = reinterpret_cast<const __half2*>(&ub);
            float wa[8], wb[8];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float2 fa = __half22float2(ha[i]), fb = __half22float2(hb[i]);
              wa[2 * i] = fa.x; wa[2 * i + 1] = fa.y;
              wb[2 * i] = fb.x; wb[2 * i + 1] = fb.y;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
              for (int r = 0; r < NR; ++r) {
                acc[m][r] = fmaf(xv[r][i], wa[i], acc[m][r]);
                acc[m + 1][r] = fmaf(xv[r][i], wb[i], acc[m + 1][r]);
              }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(ring_empty0 + 8u * st);
      ++unit;
    }
    // ---- group done: reduce over the K-slices (lanes by a transposing shuffle network, warps through smem)
    trace_ev(A, ctid, s_tr, 4);
    float* sr = s_red + (grp_idx & 1) * (NSET * MG_CONS_WARPS * 32);  // double buffered: one barrier per group
    float red[32];
#pragma unroll
    for (int set = 0; set < NSET; ++set) {
#pragma unroll
      for (int i = 0; i < 32; ++i) red[i] = 0.f;
#pragma unroll
      for (int j = 0; j < GP; ++j)
#pragma unroll
        for (int r = 0; r < NR; ++r) red[j * NR + r] = acc[set * GP + j][r];
      sr[(set * MG_CONS_WARPS + warp) * 32 + lane] = warp_transpose_reduce32(red, lane);
    }
    if (ln && grp_idx == 0) {
#pragma unroll
      for (int i = 0; i < 32; ++i) red[i] = 0.f;
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        red[r] = sx[r];
        red[16 + r] = sxx[r];
      }
      s_lnred[warp * 32 + lane] = warp_transpose_reduce32(red, lane);
    }
    ++grp_idx;
    trace_ev(A, ctid, s_tr, 5);
    cons_sync();
    trace_ev(A, ctid, s_tr, 6);
    // the last two consumer warps finish the outputs (with d_model >= 1280 they hold no K-slice, so this overlaps the
    // other warps' next group; the reduction buffer is double buffered and the next cons_sync orders its reuse)
    if (ctid >= MG_CONS - 64) {
      for (int idx = ctid - (MG_CONS - 64); idx < n_parts * NSET * 32; idx += 64) {
        const int p = idx / (NSET * 32), set = (idx >> 5) % NSET, i = idx & 31;
        const int j = i / NR, r = i - j * NR;
        const int cj = p + n_parts * (set * GP + j);
        if (j < GP && cj < nc && r < R) {
          float v = 0.f;
          for (int w = 0; w < wpp; ++w) v += sr[(set * MG_CONS_WARPS + p * wpp + w) * 32 + i];
          const int n = g0 + cj;
          if (ln) {
            float t1 = 0.f, t2 = 0.f;
            for (int w = 0; w < wpp; ++w) {
              t1 += s_lnred[w * 32 + r];
              t2 += s_lnred[w * 32 + 16 + r];
            }
            const float mean = t1 / g.K;
            const float rstd = rsqrtf(fmaxf(t2 / g.K - mean * mean, 0.f) + 1e-5f);
            v = rstd * (v - mean * (pre ? s_s2[n - lo] : __ldg(g.ln_s2 + n)));
          }
          v += pre ? s_bias[n - lo] : (g.bias != nullptr ? __ldg(g.bias + n) : 0.f);
          switch (g.epi) {
            case GV_STORE:
              g.out[static_cast<long long>(r) * g.ldo + n] = v;
              break;
            case GV_RESID: {  // residual columns are owned by this CTA for the whole pass: no global read-modify-write
              const float nv = s_xown[r * 16 + (n - lo)] + v;
              s_xown[r * 16 + (n - lo)] = nv;
              g.out[static_cast<long long>(r) * g.ldo + n] = nv;
              break;
            }
            case GV_GELU:
              g.out[static_cast<long long>(r) * g.ldo + n] = gelu_erf(v);
              break;
            case GV_QKV: {
              const int d = A.d;
              if (n < d) {
                g.out[static_cast<long long>(r) * g.ldo + n] = v;
              } else {
                const int pos = row_pos(A, r);
                __half* cache = (n < 2 * d) ? ly->kcache : ly->vcache;
                const int e = (n < 2 * d) ? n - d : n - 2 * d;
                cache[(static_cast<long long>(row_slot(A, r)) * A.t_max + pos) * d + e] = __float2half_rn(v);
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
  rg.unit = unit;
}

// ------------------------------------------------------------------ consumer: self-attention phase
// task = (row, head), one warp each.  Lane t owns key t of a 32-key block: its K row and V row are requested together (one
// L2 round trip for the whole block), the V rows are parked in shared memory (16-byte chunks XOR-swizzled by key) and the
// P.V product then runs from shared memory with lanes over the head dimension.  The step position, the ping-pong flag and
// the warp's cache-slot table are pass constants, read once at kernel start (`pos_dec`, `flipv`, `s_slot_tab`).
__device__ __noinline__ void consume_self_attn(const MegaArgs& A, const MegaLayer& ly, int ctid, uint8_t* s_scr,
                                               const unsigned short* s_slot_tab, int pos_dec, int flipv, int* s_tr) {
  const int lane = ctid & 31, warp = ctid >> 5;
  const int d = A.d, H = A.H;
  const int n_tasks = A.R * H;
  const bool pf = A.pf_len > 0;
  const uint32_t sv = smem_u32(s_scr) + warp * 4224;
  float* sp = reinterpret_cast<float*>(s_scr + warp * 4224 + 4096);
  const unsigned short* my_slots = s_slot_tab + warp * 448;
  const __half* kcache = ly.kcache;
  const __half* vcache = ly.vcache;
  trace_ev(A, ctid, s_tr, 20);
  for (int base = blockIdx.x * MG_CONS_WARPS; base < n_tasks; base += gridDim.x * MG_CONS_WARPS) {
    const int task = base + warp;
    if (task < n_tasks) {
      const bool tab = base == static_cast<int>(blockIdx.x) * MG_CONS_WARPS;
      const int r = task / H, h = task - r * H;
      const int pos = pf ? r % A.pf_len : pos_dec;
      const int own = row_slot(A, r);
      const int* indir = (flipv ? A.indir1 : A.indir0) + static_cast<long long>(r) * A.t_max;
      const float* qr = A.q + static_cast<long long>(r) * d + h * HEAD_DIM;
      float m = -INFINITY, l = 0.f, o0 = 0.f, o1 = 0.f;
      for (int t0 = 0; t0 <= pos; t0 += 32) {
        const int t = t0 + lane;
        const bool valid = t <= pos;
        int slot = own;
        if (valid && !pf && t != pos) slot = tab ? static_cast<int>(my_slots[t]) : __ldcg(indir + t);
        uint4 ku[8], vu[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) ku[i] = vu[i] = make_uint4(0u, 0u, 0u, 0u);
        if (valid) {
          const long long off = (static_cast<long long>(slot) * A.t_max + t) * d + h * HEAD_DIM;
          const uint4* kr = reinterpret_cast<const uint4*>(kcache + off);
          const uint4* vr = reinterpret_cast<const uint4*>(vcache + off);
#pragma unroll
          for (int i = 0; i < 8; ++i) ku[i] = __ldcg(kr + i);
#pragma unroll
          for (int i = 0; i < 8; ++i) vu[i] = __ldcg(vr + i);
        }
        float sc0 = 0.f, sc1 = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 qa = ldcg_f4(qr + 8 * i), qb = ldcg_f4(qr + 8 * i + 4);
          const __half2* h2 = reinterpret_cast<const __half2*>(&ku[i]);
          const float2 f0 = __half22float2(h2[0]), f1 = __half22float2(h2[1]), f2 = __half22float2(h2[2]), f3 = __half22float2(h2[3]);
          sc0 = fmaf(qa.x, f0.x, sc0); sc1 = fmaf(qa.y, f0.y, sc1);
          sc0 = fmaf(qa.z, f1.x, sc0); sc1 = fmaf(qa.w, f1.y, sc1);
          sc0 = fmaf(qb.x, f2.x, sc0); sc1 = fmaf(qb.y, f2.y, sc1);
          sc0 = fmaf(qb.z, f3.x, sc0); sc1 = fmaf(qb.w, f3.y, sc1);
        }
        const float sc = valid ? (sc0 + sc1) * 0.125f : -INFINITY;
        trace_ev(A, ctid, s_tr, 21);
#pragma unroll
        for (int i = 0; i < 8; ++i) sts128(sv + lane * 128 + ((i ^ (lane & 7)) << 4), vu[i]);
        const float mn = fmaxf(m, warp_max(sc));
        const float resc = __expf(m - mn);
        const float p = valid ? __expf(sc - mn) : 0.f;
        l = fmaf(l, resc, warp_sum(p));
        o0 *= resc;
        o1 *= resc;
        m = mn;
        sp[lane] = p;
        __syncwarp();
        trace_ev(A, ctid, s_tr, 22);
        const int nb = min(32, pos - t0 + 1);
#pragma unroll 4
        for (int tt = 0; tt < nb; ++tt) {
          const float pp = sp[tt];
          const uint32_t u = lds32(sv + tt * 128 + (((lane >> 2) ^ (tt & 7)) << 4) + ((lane & 3) << 2));
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&u));
          o0 = fmaf(pp, f.x, o0);
          o1 = fmaf(pp, f.y, o1);
        }
        __syncwarp();
      }
      trace_ev(A, ctid, s_tr, 23);
      const float inv = 1.0f / l;
      store_ctx2(A, r, h * HEAD_DIM + 2 * lane, o0 * inv, o1 * inv);
      trace_ev(A, ctid, s_tr, 24);
    }
  }
}

// ------------------------------------------------------------------ consumer: cross-attention phase
// 28 groups of 8 lanes walk the split's keys with an online softmax for all beams at once (K/V are read once for every
// beam); groups are merged by shuffles (4 per warp) and shared memory into one partial (acc[64], m, l) per beam; the
// last split of a head to arrive (atomic counter) merges the S partials into ctx.
// kOneArrive: the ring's empty barriers count ONE arrival per stage instead of one per consumer warp
// second half of a cross-attention task: the warps' partials (s_part: [warp][beam][64 acc, m, l]) are merged into the CTA's
// partial for its key split, published, and split 0 of the head merges the S partials into the attention output
template <int NB, bool kOneArrive, bool kMma>
__device__ __forceinline__ void cross_tail(const MegaArgs& A, const CrossGeom& cg, int ctid, float* s_part, unsigned tag, int* s_tr,
                                           uint32_t xbar, unsigned* x_count, int uh, int u, int h, int split, int beam,
                                           uint32_t ring_empty0, int stK, int stV) {
  float* cross_part = A.cross_part;
  trace_ev(A, ctid, s_tr, 14);
  cons_sync();
  if (kOneArrive && ctid == 0) {  // every warp has left the K / V stages
    mbar_arrive(ring_empty0 + 8u * stK);
    mbar_arrive(ring_empty0 + 8u * stV);
  }
  for (int idx = ctid; idx < beam * HEAD_DIM; idx += MG_CONS) {
    const int k = idx / HEAD_DIM, e = idx - k * HEAD_DIM;
    float mm = -INFINITY;
    for (int g = 0; g < MG_CONS_WARPS; ++g) mm = fmaxf(mm, s_part[(g * NB + k) * 66 + 64]);
    float a = 0.f, ll = 0.f;
    for (int g = 0; g < MG_CONS_WARPS; ++g) {
      const float mg = s_part[(g * NB + k) * 66 + 64];
      const float w = (mg == -INFINITY) ? 0.f : __expf(mg - mm);
      a = fmaf(w, s_part[(g * NB + k) * 66 + e], a);
      ll = fmaf(w, s_part[(g * NB + k) * 66 + 65], ll);
    }
    float* out = cross_part + (static_cast<long long>(uh) * cg.S + split) * (MAX_BEAM * 68) + k * 68;
    out[e] = a;
    if (e == 0) {
      out[64] = mm;
      out[65] = ll;
    }
  }
  // split-K fix-up without atomics or fences on the critical path: every split publishes an epoch-tagged flag (release
  // store by one thread after the CTA barrier); split 0 of the head polls the S flags (acquire) and merges the partials.
  // All other CTAs go straight on to the grid barrier.
  trace_ev(A, ctid, s_tr, 15);
  cons_sync();
  if (ctid == 0) st_release_gpu(A.cross_flags + (uh * 16 + split) * 32, tag);
  if (split == 0) {
    if (ctid < cg.S) {
      const unsigned* f = A.cross_flags + (uh * 16 + ctid) * 32;
      while (ld_acquire_gpu(f) != tag) {
      }
    }
    trace_ev(A, ctid, s_tr, 16);
    cons_sync();
    const float* pbase = cross_part + (static_cast<long long>(uh) * cg.S) * (MAX_BEAM * 68);
    // warp-MMA pass: the S partial blocks of the head are contiguous -- one bulk copy into the (now idle) merge area
    // instead of 2 x S dependent ld.global per thread
    const uint32_t pbytes = static_cast<uint32_t>(cg.S * MAX_BEAM * 68 * 4);
    const bool via_smem = kMma && pbytes <= 24576u;
    if (via_smem) {
      if (ctid == 0) {
        asm volatile("fence.proxy.async.global;" ::: "memory");
        mbar_arrive_expect_tx(xbar, pbytes);
        bulk_load_1d(smem_u32(s_part), pbase, pbytes, xbar);
      }
      mbar_wait(xbar, *x_count & 1u);
      ++*x_count;
      pbase = s_part;
    }
    // every load of the merge is issued before the first use: one round trip for the whole fix-up
    for (int idx = ctid; idx < beam * (HEAD_DIM / 2); idx += MG_CONS) {
      const int k = idx / (HEAD_DIM / 2), e = (idx - k * (HEAD_DIM / 2)) * 2;
      const float* pb = pbase + k * 68;
      float2 ml[16], pv[16];
#pragma unroll
      for (int s2 = 0; s2 < 16; ++s2) {
        ml[s2] = make_float2(-INFINITY, 0.f);
        pv[s2] = make_float2(0.f, 0.f);
        if (s2 < cg.S) {
          if (via_smem) {
            ml[s2] = *reinterpret_cast<const float2*>(pb + s2 * (MAX_BEAM * 68) + 64);
            pv[s2] = *reinterpret_cast<const float2*>(pb + s2 * (MAX_BEAM * 68) + e);
          } else {
            ml[s2] = ldcg_f2(pb + s2 * (MAX_BEAM * 68) + 64);
            pv[s2] = ldcg_f2(pb + s2 * (MAX_BEAM * 68) + e);
          }
        }
      }
      float mm = -INFINITY;
#pragma unroll
      for (int s2 = 0; s2 < 16; ++s2) mm = fmaxf(mm, ml[s2].x);
      float ax = 0.f, ay = 0.f, ll = 0.f;
#pragma unroll
      for (int s2 = 0; s2 < 16; ++s2) {
        const float w = (ml[s2].x == -INFINITY) ? 0.f : __expf(ml[s2].x - mm);
        ax = fmaf(w, pv[s2].x, ax);
        ay = fmaf(w, pv[s2].y, ay);
        ll = fmaf(w, ml[s2].y, ll);
      }
      const float inv = 1.f / ll;
      store_ctx2(A, u * beam + k, h * HEAD_DIM + e, ax * inv, ay * inv);
    }
  }
  trace_ev(A, ctid, s_tr, 17);
  cons_sync();
}

template <int NB, bool kOneArrive = false, int NS = MG_NSTAGE, bool kMma = false>
__device__ __forceinline__ void consume_cross_impl(Ring& rg, const MegaArgs& A, int ctid, float* s_part, unsigned tag, int* s_tr,
                                                uint32_t xbar = 0, unsigned* x_count = nullptr) {
  const int grp = ctid >> 3, gl = ctid & 7;
  constexpr int NGRP = MG_CONS / 8;  // 28
  const int d = A.d, beam = A.beam, H = A.H;
  const float* qbase = A.q;
  float* cross_part = A.cross_part;
  const uint32_t ring_data0 = rg.data0, ring_full0 = rg.full0, ring_empty0 = rg.empty0;
  unsigned unit = rg.unit;
  const unsigned gmask = 0xFFu << (ctid & 24);
  const CrossGeom cg = cross_geom(A.n_utt, H);
  trace_ev(A, ctid, s_tr, 10);
  for (int task = blockIdx.x; task < cg.n_tasks; task += gridDim.x) {
    const int split = task % cg.S, uh = task / cg.S;
    const int u = uh / H, h = uh - u * H;
    const int t0 = split * cg.KS;
    int nk = min(cg.KS, T_ENC - t0);  // keys >= 1500 (padding rows) are never touched
    if (nk < 0) nk = 0;
    const int stK = unit % NS, stV = (unit + 1) % NS;
    float qv[NB][8];
#pragma unroll
    for (int k = 0; k < NB; ++k) {
#pragma unroll
      for (int i = 0; i < 8; ++i) qv[k][i] = 0.f;
      if (k < beam) {
        const float* qr = qbase + static_cast<long long>(u * beam + k) * d + h * HEAD_DIM + gl * 8;
        const float4 a0 = ldcg_f4(qr), a1 = ldcg_f4(qr + 4);
        qv[k][0] = a0.x * 0.125f; qv[k][1] = a0.y * 0.125f; qv[k][2] = a0.z * 0.125f; qv[k][3] = a0.w * 0.125f;
        qv[k][4] = a1.x * 0.125f; qv[k][5] = a1.y * 0.125f; qv[k][6] = a1.z * 0.125f; qv[k][7] = a1.w * 0.125f;
      }
    }
    float m[NB], l[NB], acc[NB][8];
#pragma unroll
    for (int k = 0; k < NB; ++k) {
      m[k] = -INFINITY;
      l[k] = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[k][i] = 0.f;
    }
    trace_ev(A, ctid, s_tr, 11);
    mbar_wait(ring_full0 + 8u * stK, (unit / NS) & 1u);
    mbar_wait(ring_full0 + 8u * stV, ((unit + 1) / NS) & 1u);
    const uint32_t sK = ring_data0 + stK * MG_STAGE_BYTES, sV = ring_data0 + stV * MG_STAGE_BYTES;
    trace_ev(A, ctid, s_tr, 12);
#pragma unroll 1
    for (int tl = grp; tl < nk; tl += 2 * NGRP) {
      // two keys per step with one joint running-max update: shorter dependency chains, 3 exps and 3 FMAs per pair
      const bool hasb = tl + NGRP < nk;
      const int tb = hasb ? tl + NGRP : tl;
      const uint4 kua = lds128(sK + tl * (HEAD_DIM * 2) + gl * 16), kub = lds128(sK + tb * (HEAD_DIM * 2) + gl * 16);
      const uint4 vua = lds128(sV + tl * (HEAD_DIM * 2) + gl * 16), vub = lds128(sV + tb * (HEAD_DIM * 2) + gl * 16);
      float sa[NB], sb[NB];
#pragma unroll
      for (int k = 0; k < NB; ++k) sa[k] = sb[k] = 0.f;
      {
        const __half2* ka2 = reinterpret_cast<const __half2*>(&kua);
        const __half2* kb2 = reinterpret_cast<const __half2*>(&kub);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 fa = __half22float2(ka2[i]), fb = __half22float2(kb2[i]);
#pragma unroll
          for (int k = 0; k < NB; ++k) {
            sa[k] = fmaf(qv[k][2 * i], fa.x, sa[k]);
            sb[k] = fmaf(qv[k][2 * i], fb.x, sb[k]);
            sa[k] = fmaf(qv[k][2 * i + 1], fa.y, sa[k]);
            sb[k] = fmaf(qv[k][2 * i + 1], fb.y, sb[k]);
          }
        }
      }
      float vfa[8], vfb[8];
      {
        const __half2* va2 = reinterpret_cast<const __half2*>(&vua);
        const __half2* vb2 = reinterpret_cast<const __half2*>(&vub);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 fa = __half22float2(va2[i]), fb = __half22float2(vb2[i]);
          vfa[2 * i] = fa.x; vfa[2 * i + 1] = fa.y;
          vfb[2 * i] = fb.x; vfb[2 * i + 1] = fb.y;
        }
      }
#pragma unroll
      for (int k = 0; k < NB; ++k) {
        float xa = sa[k], xb = sb[k];
        xa += __shfl_xor_sync(gmask, xa, 1);
        xb += __shfl_xor_sync(gmask, xb, 1);
        xa += __shfl_xor_sync(gmask, xa, 2);
        xb += __shfl_xor_sync(gmask, xb, 2);
        xa += __shfl_xor_sync(gmask, xa, 4);
        xb += __shfl_xor_sync(gmask, xb, 4);
        if (!hasb) xb = -INFINITY;
        const float mn = fmaxf(m[k], fmaxf(xa, xb));
        const float al = __expf(m[k] - mn), pa = __expf(xa - mn), pb = __expf(xb - mn);
        l[k] = fmaf(l[k], al, pa + pb);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[k][i] = fmaf(acc[k][i], al, fmaf(pa, vfa[i], pb * vfb[i]));
        m[k] = mn;
      }
    }
    trace_ev(A, ctid, s_tr, 13);
    __syncwarp();
    if (!kOneArrive && (ctid & 31) == 0) {
      mbar_arrive(ring_empty0 + 8u * stK);
      mbar_arrive(ring_empty0 + 8u * stV);
    }
    unit += 2;
    // merge: the 4 groups of a warp with shuffles (lanes l, l^8, l^16 hold the same dims), then the warps through smem
#pragma unroll
    for (int k = 0; k < NB; ++k) {
#pragma unroll
      for (int off = 8; off <= 16; off <<= 1) {
        const float mo = __shfl_xor_sync(0xffffffffu, m[k], off);
        const float lo_ = __shfl_xor_sync(0xffffffffu, l[k], off);
        const float mn = fmaxf(m[k], mo);
        const float wa = (m[k] == -INFINITY) ? 0.f : __expf(m[k] - mn);
        const float wb = (mo == -INFINITY) ? 0.f : __expf(mo - mn);
        l[k] = l[k] * wa + lo_ * wb;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float ao = __shfl_xor_sync(0xffffffffu, acc[k][i], off);
          acc[k][i] = acc[k][i] * wa + ao * wb;
        }
        m[k] = mn;
      }
      if ((ctid & 31) < 8) {
        float* dst = s_part + ((ctid >> 5) * NB + k) * 66;
#pragma unroll
        for (int i = 0; i < 8; ++i) dst[gl * 8 + i] = acc[k][i];
        if (gl == 0) {
          dst[64] = m[k];
          dst[65] = l[k];
        }
      }
    }
    cross_tail<NB, kOneArrive, kMma>(A, cg, ctid, s_part, tag, s_tr, xbar, x_count, uh, u, h, split, beam, ring_empty0, stK, stV);
  }
  rg.unit = unit;
}

template <int NB>
__device__ __noinline__ void consume_cross(Ring& rg, const MegaArgs& A, int ctid, float* s_part, unsigned tag, int* s_tr) {
  consume_cross_impl<NB, false, MG_NSTAGE, false>(rg, A, ctid, s_part, tag, s_tr);
}

template <int NR>
__global__ void __launch_bounds__(MG_THREADS, 1) dec_pass_kernel(const MegaArgs A) {
  if (A.pf_len == 0 && A.st->all_done) return;  // a step enqueued ahead of the host's poll (every thread of every CTA leaves)
  extern __shared__ __align__(1024) uint8_t mg_smem[];
  uint8_t* ring_data = mg_smem;
  uint64_t* bars = reinterpret_cast<uint64_t*>(mg_smem + MG_NSTAGE * MG_STAGE_BYTES);
  float* s_red = reinterpret_cast<float*>(mg_smem + MG_NSTAGE * MG_STAGE_BYTES + 1024);
  float* s_stat = s_red + MG_RED_FLOATS;  // 1056 floats: [0,256) unused, bias, s2, own residual columns, flags
  float* s_part = s_stat + 1056;  // [warps][NB][66] for the cross-attention merge; also self-attention scratch
  unsigned short* s_slot_tab = reinterpret_cast<unsigned short*>(reinterpret_cast<uint8_t*>(s_part) + MG_SCRATCH);
  MegaLayer* s_ly = reinterpret_cast<MegaLayer*>(reinterpret_cast<uint8_t*>(s_slot_tab) + MG_SLOT_BYTES);  // [2] at 512 B
  Ring rg;
  rg.data = ring_data;
  rg.data0 = smem_u32(ring_data);
  rg.full0 = smem_u32(bars);
  rg.empty0 = rg.full0 + 8 * MG_NSTAGE;
  rg.unit = 0;
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < MG_NSTAGE; ++s) {
      mbar_init(rg.full(s), 1);
      mbar_init(rg.empty(s), MG_CONS_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int L = A.n_layers;

  if (tid >= MG_CONS) {
    // ============================ producer: the static weight / KV stream of this CTA
    if (tid == MG_CONS) {
      for (int l = 0; l < L; ++l) {
        const MegaLayer& ly = A.layers[l];
        produce_gemv(rg, ly.qkv, mg_gp(NR) * mg_nset(NR));
        produce_gemv(rg, ly.o, mg_gp(NR) * mg_nset(NR));
        produce_gemv(rg, ly.cq, mg_gp(NR) * mg_nset(NR));
        produce_cross(rg, A, ly);
        produce_gemv(rg, ly.co, mg_gp(NR) * mg_nset(NR));
        produce_gemv(rg, ly.fc1, mg_gp(NR) * mg_nset(NR));
        produce_gemv(rg, ly.fc2, mg_gp(NR) * mg_nset(NR));
      }
      if (A.with_logits) produce_gemv(rg, A.vocab, mg_gp(NR) * mg_nset(NR));
    }
    return;
  }
  // ============================== consumers
  const int ctid = tid;
  unsigned epoch = *A.epoch_base;  // flags hold the epoch of the previous launch
  const unsigned epoch0 = epoch;
  int* s_tr0 = reinterpret_cast<int*>(s_stat + 912);  // [912, 1056): event trace
  if (ctid == 0) s_tr0[0] = -1;
  if (A.trace != nullptr && blockIdx.x == 0 && ctid == 0) A.trace[0] = globaltimer_ns();
  // layer descriptors travel to shared memory one layer ahead (cp.async), so no phase starts with a global round trip
  auto prefetch_layer = [&](int l) {
    if (ctid < static_cast<int>(sizeof(MegaLayer) / 16))
      cp_async16(smem_u32(reinterpret_cast<uint8_t*>(s_ly) + (l & 1) * MG_LY_STRIDE) + ctid * 16,
                 reinterpret_cast<const uint8_t*>(A.layers + l) + ctid * 16);
  };
  if (L > 0) prefetch_layer(0);
  // pass constants: step position, indirection ping-pong flag, and the cache slots of this warp's self-attention task
  const int pos_dec = A.pf_len > 0 ? 0 : A.st->pos;
  const int flipv = *A.flip;
  if (A.pf_len == 0) {
    const int task = blockIdx.x * MG_CONS_WARPS + (ctid >> 5);
    if (task < A.R * A.H) {
      const int* indir = (flipv ? A.indir1 : A.indir0) + static_cast<long long>(task / A.H) * A.t_max;
      for (int t = ctid & 31; t < pos_dec; t += 32) s_slot_tab[(ctid >> 5) * 448 + t] = static_cast<unsigned short>(indir[t]);
    }
  }
  cp_async_wait_all();
  // phase 0: token + positional embedding; every CTA produces (and keeps) the residual-stream columns it owns
  {
    int lo, hi;
    cta_cols(A.d, lo, hi);
    float* s_xown = s_stat + 784;
    for (int idx = ctid; idx < A.R * (hi - lo); idx += MG_CONS) {
      const int r = idx / (hi - lo), c = idx - r * (hi - lo);
      const float v = __half2float(A.tok_emb[static_cast<long long>(row_token(A, r)) * A.d + lo + c]) +
                      A.pos_emb[static_cast<long long>(row_pos(A, r)) * A.d + lo + c];
      s_xown[r * 16 + c] = v;
      A.x[static_cast<long long>(r) * A.d + lo + c] = v;
    }
  }
  grid_barrier(A, epoch, ctid, epoch0);
  for (int l = 0; l < L; ++l) {
    const MegaLayer& ly = *reinterpret_cast<const MegaLayer*>(reinterpret_cast<const uint8_t*>(s_ly) + (l & 1) * MG_LY_STRIDE);
    if (l + 1 < L) prefetch_layer(l + 1);  // the other buffer was last read in layer l - 1
    trace_open(A, ctid, s_tr0, l);
    consume_gemv<NR>(rg, A, ly.qkv, &ly, ctid, s_red, s_stat);
    grid_barrier(A, epoch, ctid, epoch0);
    consume_self_attn(A, ly, ctid, reinterpret_cast<uint8_t*>(s_part), s_slot_tab, pos_dec, flipv, s_tr0);
    grid_barrier(A, epoch, ctid, epoch0);
    consume_gemv<NR>(rg, A, ly.o, &ly, ctid, s_red, s_stat);
    grid_barrier(A, epoch, ctid, epoch0);
    consume_gemv<NR>(rg, A, ly.cq, &ly, ctid, s_red, s_stat);
    grid_barrier(A, epoch, ctid, epoch0);
    consume_cross<NR>(rg, A, ctid, s_part, epoch + 1, s_tr0);  // beam <= rows <= NR; tag = a value unique to this phase
    grid_barrier(A, epoch, ctid, epoch0);
    consume_gemv<NR>(rg, A, ly.co, &ly, ctid, s_red, s_stat);
    grid_barrier(A, epoch, ctid, epoch0);
    consume_gemv<NR>(rg, A, ly.fc1, &ly, ctid, s_red, s_stat);
    grid_barrier(A, epoch, ctid, epoch0);
    consume_gemv<NR>(rg, A, ly.fc2, &ly, ctid, s_red, s_stat);
    cp_async_wait_all();  // next layer's descriptor has landed; the barrier's CTA sync publishes it
    grid_barrier(A, epoch, ctid, epoch0);
  }
  if (A.with_logits) consume_gemv<NR>(rg, A, A.vocab, nullptr, ctid, s_red, s_stat);
  // publish the final epoch for the next launch (every CTA leaves the same value behind)
  grid_barrier(A, epoch, ctid, epoch0);
  trace_dump(A, ctid, s_tr0);
  if (blockIdx.x == 0 && ctid == 0) {
    *A.epoch_base = epoch;
    A.epoch_base[8] = epoch * gridDim.x;  // keeps the counter of the atomic barrier mode in step whatever mode ran
  }
}


// =====================================================================================================================
// Warp-MMA variant of the pass: the six GEMV phases of a layer and the vocabulary projection run on the warp-level tensor
// path (mma.sync.m16n8k16, fp16 x fp16 -> fp32): the CTA's weight rows are the MMA's M (16-row tiles), the <= 8 activation
// rows its N, K is split over the 7 consumer warps and their partial tiles are summed through shared memory.
// Why not wgmma here (it is what the encoder, the batched pass and the cross-attention of the batched pass use): at N = 8
// a warpgroup MMA is one 64 x 8 x 16 instruction for four warps, and this pass splits K over 7 consumer warps that each
// work on their own 16-row tiles; the warp MMA fits that split directly (scripts/diag_gemv_tc.py times the wgmma GEMV
// at the same shapes for comparison).  18 (k-block, m-tile) items of 4 HMMAs each per warp cover the QKV phase.  What disappears against the SIMT pass: the
// fp32 FMA loop over the weight stage and the transposing shuffle reductions.  What stays: the
// producer thread and its static weight schedule (2-D TMA boxes, 128-byte swizzle, straight from the row-major W -- the
// swizzle is what makes ldmatrix conflict-free), the grid barrier between phases, the attention phases, LayerNorm folded
// into the epilogue, residual columns owned by the CTA.  Columns are dealt to the CTAs in whole octets (8-row swizzle
// atoms), so no CTA streams a neighbour's weight rows.
// Activations are rounded to fp16 when they become the B operand (the encoder and the batched pass do the same).
// =====================================================================================================================
// shared-memory plan of the warp-MMA kernel: ring | B operand (aliased by the attention scratch) | partial tiles | barriers,
// statistics, trace cursor, owned residual columns | cache-slot tables | layer descriptors | phase geometry
constexpr int FUSED_B_OFF = 36864;  // fused cross phase: its B operand image inside s_b, above the merge area and the statistic shares
template <int NR>
struct MmaSmem {
  static constexpr int NS = NR <= 5 ? 4 : 3;                 // ring stages: a whole next phase's weights fit ahead of the consumers
  static constexpr int B_BYTES = (5120 / 64) * NR * 128;     // B operand image of the largest K (fc2): [K/64][R][128 B]
  static constexpr int B_MIN = FUSED_B_OFF + 20 * NR * 128;  // fused cross phase: merge area | statistics | B operand
  static constexpr int B_ALLOC = B_BYTES > B_MIN ? (B_BYTES > MG_SCRATCH ? B_BYTES : MG_SCRATCH) : (B_MIN > MG_SCRATCH ? B_MIN : MG_SCRATCH);
  static constexpr int OFF_B = NS * MG_STAGE_BYTES;          // (an m-tile's 16-row read may run 1 KB past its box: harmless)
  static constexpr int OFF_PART = OFF_B + B_ALLOC;
  static constexpr int PART_BYTES = MG_CONS_WARPS * 8 * 68 * 4;
  static constexpr int OFF_BARS = OFF_PART + PART_BYTES;
  static constexpr int OFF_STAT = OFF_BARS + 256;            // 1056 floats, same map as the SIMT kernel's s_stat
  static constexpr int OFF_SLOT = OFF_STAT + 4224;
  static constexpr int OFF_LY = OFF_SLOT + MG_SLOT_BYTES;
  static constexpr int OFF_GEOM = OFF_LY + MG_LY_BYTES;
  static constexpr int TOTAL = OFF_GEOM + 5 * 64;
  static constexpr int STAT_OFF = 24576;                     // row-statistics shares land behind the image of a K <= 1280 phase
  static_assert(TOTAL <= 232448, "warp-MMA decoder pass: shared memory");
  static_assert(20 * NR * 128 <= STAT_OFF && STAT_OFF + 160 * NR * 8 <= FUSED_B_OFF && FUSED_B_OFF + 20 * NR * 128 <= B_ALLOC,
                "statistics landing zone / fused-phase B operand");
};
constexpr int MM_GROUP_ROWS = 64;       // weight rows per accumulation group (4 m-tiles)
constexpr int MM_PART_LD = 68;          // partial tiles [warp][8 rows][68]: conflict-free fragment stores

// columns of a GEMV phase owned by this CTA: N / grid each, the first N % grid CTAs one more (row granularity: with whole
// octets some CTAs would own twice the columns of the others and close every d-wide phase late); ring units of a group of `rows` weight rows: as many 64-wide k-blocks as
// fit a stage, evenly sized.  Computed once per kernel for the five
// GEMV shapes (qkv, d x d, fc1, fc2, vocabulary): at one warp per scheduler every instruction on a phase's critical path
// counts, and these integer divisions would otherwise sit on it in every phase.
struct MmaGeom {
  int lo, hi, rows_pad, n_full, tail;
  int units_full, kbu_full, units_tail, kbu_tail, pad[7];
};
static_assert(sizeof(MmaGeom) == 64, "geometry table stride");
__device__ __forceinline__ void mma_units(int rows, int kblocks, int& units, int& kbu) {
  const int max_kbu = MG_STAGE_BYTES / (rows * 128);
  units = (kblocks + max_kbu - 1) / max_kbu;
  kbu = (kblocks + units - 1) / units;
}
__device__ __forceinline__ MmaGeom mma_geom(int N, int K) {
  MmaGeom m;
  const int G = static_cast<int>(gridDim.x), b = static_cast<int>(blockIdx.x);
  const int base = N / G, rem = N - base * G;
  m.lo = b * base + min(b, rem);
  m.rows_pad = base + (b < rem ? 1 : 0);
  m.hi = m.lo + m.rows_pad;
  m.n_full = m.rows_pad / MM_GROUP_ROWS;
  m.tail = m.rows_pad - m.n_full * MM_GROUP_ROWS;
  m.units_full = m.kbu_full = m.units_tail = m.kbu_tail = 0;
  if (m.n_full > 0) mma_units(MM_GROUP_ROWS, K / 64, m.units_full, m.kbu_full);
  if (m.tail > 0) mma_units(m.tail, K / 64, m.units_tail, m.kbu_tail);
  return m;
}

template <int NS>
__device__ __forceinline__ void produce_gemv_mma(Ring& rg, const MegaGemv& g, const MmaGeom* s_geom, int dbg) {
  const MmaGeom mg = s_geom[g.shape];
  const int n_groups = mg.n_full + (mg.tail ? 1 : 0);
  const int kblocks = g.K / 64;
  const uint64_t pol = l2_policy_evict_first();
  for (int gi = 0; gi < n_groups; ++gi) {
    const bool full = gi < mg.n_full;
    const int rows = full ? MM_GROUP_ROWS : mg.tail;
    const int units = full ? mg.units_full : mg.units_tail, kbu = full ? mg.kbu_full : mg.kbu_tail;
    // g.w is the warp-MMA image of W (mma_image_kernel): the group's k-blocks are contiguous [k-block][rows][128 B swizzled]
    const __half* base = g.w + static_cast<long long>(mg.lo + gi * MM_GROUP_ROWS) * g.K;
    for (int u = 0; u < units; ++u) {
      const int kb0 = u * kbu, nkb = min(kbu, kblocks - kb0);
      const int st = rg.unit % NS;
      mbar_wait(rg.empty(st), ((rg.unit / NS) & 1u) ^ 1u);
      uint32_t bytes = static_cast<uint32_t>(nkb * rows * 128);
      if (dbg & 2) bytes = (bytes >> 2) & ~15u;  // diagnostics: a quarter of the weight traffic (results are garbage)
      mbar_arrive_expect_tx(rg.full(st), bytes);
      bulk_load_1d_hint(rg.data0 + st * MG_STAGE_BYTES, base + static_cast<long long>(kb0) * rows * 64, bytes, rg.full(st), pol);
      ++rg.unit;
    }
  }
}

// New residual-stream value of (row r, column n) leaves its owner CTA three ways: fp32 into `x` (debug / other passes),
// fp16 times the NEXT LayerNorm's gain into the exchange image the next LN-GEMV phase bulk-loads as its B operand, and as
// this CTA's share of the row's LayerNorm statistics (sum, sum of squares over its <= 16 columns) -- the consumers add the
// per-CTA shares in a fixed order, so the statistics are deterministic and nobody re-reads the fp32 row.
// Thread mapping: 16 consecutive lanes = one row; every lane of the warp must call (shuffles).
__device__ __forceinline__ void publish_resid(const MegaArgs& A, int r, int n, bool valid, float nv, float gain, int lane) {
  float s1 = valid ? nv : 0.f, s2 = valid ? nv * nv : 0.f;
#pragma unroll
  for (int off = 8; off >= 1; off >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, off);
    s2 += __shfl_xor_sync(0xffffffffu, s2, off);
  }
  if (valid) {
    A.x[static_cast<long long>(r) * A.d + n] = nv;
    A.xn16[act16_off(A.R, r, n)] = __float2half_rn(nv * gain);
  }
  if ((lane & 15) == 0 && r < A.R) *reinterpret_cast<float2*>(A.xstat + (static_cast<long long>(blockIdx.x) * A.R + r) * 2) = make_float2(s1, s2);
}

// this warp's k-blocks of one ring unit (every 7th, starting at kbi): NMT m-tiles x 4 k-steps of ldmatrix.x4 + HMMA each,
// branch- and predicate-free.  a_kb / b_kb: this lane's addresses for k-block kbi (A row of the swizzled box; B row with
// the lane's row swizzle folded in), sw[ks]: the lane's swizzled 16-byte chunk of k-step ks.
template <int NMT>
__device__ __forceinline__ void mma_unit(float (&acc)[4][4], uint32_t a_kb, uint32_t a_step, uint32_t b_kb, uint32_t b_step,
                                         int n_it, const uint32_t (&sw)[4], uint32_t b_plane) {
  // two k-blocks per trip into two accumulator sets: the second block's loads are in flight under the first block's
  // HMMA chain (one warp per scheduler: a trip's latency chain is LDS -> ldmatrix -> 4 dependent HMMAs)
  float acc2[NMT][4];
#pragma unroll
  for (int m = 0; m < NMT; ++m)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc2[m][i] = 0.f;
  int it = 0;
#pragma unroll 1
  for (; it + 1 < n_it; it += 2, a_kb += 2 * a_step, b_kb += 2 * b_step) {
    const uint4 p01 = lds128(b_kb), p23 = lds128(b_kb + b_plane);
    const uint4 q01 = lds128(b_kb + b_step), q23 = lds128(b_kb + b_step + b_plane);
    const uint32_t bf[8] = {p01.x, p01.y, p01.z, p01.w, p23.x, p23.y, p23.z, p23.w};
    const uint32_t bg[8] = {q01.x, q01.y, q01.z, q01.w, q23.x, q23.y, q23.z, q23.w};
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t af[NMT][4], ag[NMT][4];
#pragma unroll
      for (int m = 0; m < NMT; ++m) {
        ldmatrix_x4(a_kb + sw[ks] + m * 2048, af[m]);
        ldmatrix_x4(a_kb + a_step + sw[ks] + m * 2048, ag[m]);
      }
#pragma unroll
      for (int m = 0; m < NMT; ++m) {
        mma_m16n8k16(acc[m], af[m], bf[2 * ks], bf[2 * ks + 1]);
        mma_m16n8k16(acc2[m], ag[m], bg[2 * ks], bg[2 * ks + 1]);
      }
    }
  }
  if (it < n_it) {
    const uint4 b01 = lds128(b_kb), b23 = lds128(b_kb + b_plane);  // {b0, b1} of k-steps 0, 1 | 2, 3 (fragment-major image)
    const uint32_t bf[8] = {b01.x, b01.y, b01.z, b01.w, b23.x, b23.y, b23.z, b23.w};
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t af[NMT][4];
#pragma unroll
      for (int m = 0; m < NMT; ++m) ldmatrix_x4(a_kb + sw[ks] + m * 2048, af[m]);
#pragma unroll
      for (int m = 0; m < NMT; ++m) mma_m16n8k16(acc[m], af[m], bf[2 * ks], bf[2 * ks + 1]);
    }
  }
#pragma unroll
  for (int m = 0; m < NMT; ++m)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[m][i] += acc2[m][i];
}

// ------------------------------------------------------------------ warp-MMA pass: self-attention phase
// task = (row, head), one warp each; task i of CTA b is  i * grid + b  (warps 0, 1 take them alternately), so at 5 rows x 20
// heads 100 SMs work on one task each instead of 15 SMs on seven.  Per 32-key block: the K and V rows of the beam's cache
// slots are gathered into shared memory with cp.async (16 bytes per lane, 8 lanes per row, chunks XOR-swizzled by the key so
// that ldmatrix is conflict-free), the scores are one row of a 16 x 32 HMMA tile (rows 1..15 are zero), the probabilities
// stay in registers as the A operand of O += P V (V through ldmatrix.trans).  The query arrives as fp16, pre-scaled, in the
// [head][row][64] exchange layout of the QKV epilogue.
constexpr int SA_WARPS = 2;
__device__ __forceinline__ void consume_self_attn_mma(const MegaArgs& A, const MegaLayer& ly, int ctid, uint8_t* s_scr,
                                                   const unsigned short* s_slot_tab, int pos_dec, int flipv, int* s_tr) {
  const int lane = ctid & 31, warp = ctid >> 5;
  const int d = A.d, H = A.H, G = static_cast<int>(gridDim.x);
  const int n_tasks = A.R * H;
  const bool pf = A.pf_len > 0;
  trace_ev(A, ctid, s_tr, 20);
  if (warp >= SA_WARPS) return;
  const uint32_t sK = smem_u32(s_scr) + warp * 8192, sV = sK + 4096;
  const unsigned short* my_slots = s_slot_tab + warp * 448;
  const __half* kcache = ly.kcache;
  const __half* vcache = ly.vcache;
  const int gq = lane >> 2, tq = lane & 3;
  const int ld_key = lane >> 3, ld_c = lane & 7;  // gather: lane covers chunk ld_c of keys ld_key, ld_key + 4, ...
  const uint32_t lm_off = static_cast<uint32_t>(((lane & 7) + ((lane >> 3) & 1) * 8) * 128);  // ldmatrix row of this lane
  const int lm_c = lane >> 4;
  for (int i = warp; i * G + static_cast<int>(blockIdx.x) < n_tasks; i += SA_WARPS) {
    const int task = i * G + static_cast<int>(blockIdx.x);
    const bool tab = i == warp;  // the warp's first task: its cache-slot table was staged at kernel start
    const int r = task / H, h = task - r * H;
    const int pos = pf ? r % A.pf_len : pos_dec;
    const int own = row_slot(A, r);
    const int* indir = (flipv ? A.indir1 : A.indir0) + static_cast<long long>(r) * A.t_max;
    // query row -> A fragments (row 0 of the tile: lanes 0..3)
    uint32_t aq[4][2];
    {
      const __half* qr = A.q16 + (static_cast<long long>(h) * A.R + r) * HEAD_DIM + 2 * tq;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        aq[ks][0] = gq == 0 ? __ldcg(reinterpret_cast<const unsigned*>(qr + 16 * ks)) : 0u;
        aq[ks][1] = gq == 0 ? __ldcg(reinterpret_cast<const unsigned*>(qr + 16 * ks + 8)) : 0u;
      }
    }
    float m_run = -INFINITY, l_run = 0.f;
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) o[j][q] = 0.f;
    for (int t0 = 0; t0 <= pos; t0 += 32) {
      // ---- gather 32 keys (positions beyond `pos` re-read position `pos`: finite data, masked below)
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int key = it * 4 + ld_key;
        const int t = min(t0 + key, pos);
        int slot = own;
        if (!pf && t != pos) slot = tab ? static_cast<int>(my_slots[t]) : __ldcg(indir + t);
        const long long off = (static_cast<long long>(slot) * A.t_max + t) * d + h * HEAD_DIM + ld_c * 8;
        const uint32_t dst = key * 128 + ((ld_c ^ (key & 7)) << 4);
        cp_async16(sK + dst, kcache + off);
        cp_async16(sV + dst, vcache + off);
      }
      cp_async_wait_all();
      __syncwarp();
      trace_ev(A, ctid, s_tr, 21);
      // ---- scores: 4 tiles of 8 keys x 4 k-steps of 16 dims
      float sc[4][4];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) sc[nt][q] = 0.f;
#pragma unroll
      for (int kq = 0; kq < 4; ++kq) {
        const uint32_t a4[4] = {aq[kq][0], 0u, aq[kq][1], 0u};
#pragma unroll
        for (int half = 0; half < 2; ++half) {  // keys 16 half .. 16 half + 15
          uint32_t kf[4];
          ldmatrix_x4(sK + half * 2048 + lm_off + (((2 * kq + lm_c) ^ (lane & 7)) << 4), kf);
          mma_m16n8k16(sc[2 * half], a4, kf[0], kf[2]);
          mma_m16n8k16(sc[2 * half + 1], a4, kf[1], kf[3]);
        }
      }
      // ---- online softmax of tile row 0 (lanes 0..3 hold keys 8 nt + 2 tq, + 1)
      float sv[8];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int k0 = t0 + nt * 8 + 2 * tq;
        sv[2 * nt] = k0 <= pos ? sc[nt][0] : -INFINITY;
        sv[2 * nt + 1] = k0 + 1 <= pos ? sc[nt][1] : -INFINITY;
      }
      float mx = sv[0];
#pragma unroll
      for (int q = 1; q < 8; ++q) mx = fmaxf(mx, sv[q]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m_run, mx);
      const float al = __expf(m_run - mn);
      float pr[8], rs = 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        pr[q] = gq == 0 ? __expf(sv[q] - mn) : 0.f;  // rows 1..15 of the tile carry nothing
        rs += pr[q];
      }
      rs += __shfl_xor_sync(0xffffffffu, rs, 1);
      rs += __shfl_xor_sync(0xffffffffu, rs, 2);
      l_run = fmaf(l_run, al, rs);
      m_run = mn;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j][0] *= al;
        o[j][1] *= al;
      }
      // ---- O += P V: 2 k-steps of 16 keys x 8 tiles of 8 dims
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        __half2 h01 = __floats2half2_rn(pr[4 * kk], pr[4 * kk + 1]), h23 = __floats2half2_rn(pr[4 * kk + 2], pr[4 * kk + 3]);
        const uint32_t pa[4] = {*reinterpret_cast<uint32_t*>(&h01), 0u, *reinterpret_cast<uint32_t*>(&h23), 0u};
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {
          uint32_t vf[4];
          ldmatrix_x4_trans(sV + kk * 2048 + lm_off + (((2 * jp + lm_c) ^ (lane & 7)) << 4), vf);
          mma_m16n8k16(o[2 * jp], pa, vf[0], vf[1]);
          mma_m16n8k16(o[2 * jp + 1], pa, vf[2], vf[3]);
        }
      }
      __syncwarp();  // the next block's gather overwrites the rows
      trace_ev(A, ctid, s_tr, 22);
    }
    if (gq == 0) {
      const float inv = 1.0f / l_run;
#pragma unroll
      for (int j = 0; j < 8; ++j) store_ctx2(A, r, h * HEAD_DIM + 8 * j + 2 * tq, o[j][0] * inv, o[j][1] * inv);
    }
    trace_ev(A, ctid, s_tr, 24);
  }
}

// grid barrier of the warp-MMA pass (shared counter: one release-add per CTA, thread 0 spins).  The thread that sees the
// barrier open issues the NEXT phase's activation reload at once (bulk copies onto `xbar`): the copy is the first link of
// every phase's dependency chain, so it should not wait for the CTA-wide sync, the call and the descriptor loads.
struct Reload {
  const void* src = nullptr;   // fp16 exchange image -> s_b + dst_off
  uint32_t bytes = 0, dst_off = 0;
  const void* src2 = nullptr;  // per-CTA statistic shares -> s_b + stat_off
  uint32_t bytes2 = 0;
};
__device__ __forceinline__ void grid_barrier_mma(const MegaArgs& A, unsigned& epoch, int ctid, unsigned epoch0, Reload rl, uint32_t s_b_addr,
                                              uint32_t stat_off, uint32_t xbar, int* s_tr) {
  trace_ev(A, ctid, s_tr, 30);
  if (A.trace != nullptr && ctid == 0) {
    const unsigned long long t = globaltimer_ns();
    if (blockIdx.x == 0) A.trace[2 * (epoch - epoch0) + 1] = t;
    if (epoch - epoch0 < 264u) A.trace[2048 + blockIdx.x * 264 + (epoch - epoch0)] = t;  // arrival of every CTA at every barrier
  }
  cons_sync();
  trace_ev(A, ctid, s_tr, 31);
  ++epoch;
  if (ctid == 0) {
    unsigned* counter = A.epoch_base + 8;
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
    trace_ev(A, ctid, s_tr, 32);
    const unsigned target = epoch * gridDim.x;
    while (static_cast<int>(ld_acquire_gpu(counter) - target) < 0) {
    }
    trace_ev(A, ctid, s_tr, 33);
    if (rl.bytes != 0) {
      asm volatile("fence.proxy.async.global;" ::: "memory");  // other CTAs' generic-proxy stores (ordered by the barrier) -> async-proxy read
      mbar_arrive_expect_tx(xbar, rl.bytes + rl.bytes2);
      bulk_load_1d(s_b_addr + rl.dst_off, rl.src, rl.bytes, xbar);
      if (rl.bytes2 != 0) bulk_load_1d(s_b_addr + stat_off, rl.src2, rl.bytes2, xbar);
    }
  }
  cons_sync();
  if (A.trace != nullptr && blockIdx.x == 0 && ctid == 0) A.trace[2 * (epoch - epoch0)] = globaltimer_ns();
}
// reload of a GEMV phase: its input image, plus the statistic shares when it carries a LayerNorm
__device__ __forceinline__ Reload gemv_reload(const MegaArgs& A, const MegaGemv& g, const MmaGeom* s_geom) {
  Reload rl;
  if (s_geom[g.shape].rows_pad != 0) {
    rl.src = g.x16;
    rl.bytes = static_cast<uint32_t>((g.K / 64) * A.R * 128);
    if (g.ln_s2 != nullptr) {
      rl.src2 = A.xstat;
      rl.bytes2 = static_cast<uint32_t>(gridDim.x * A.R * 8);
    }
  }
  return rl;
}


template <int NR>
__device__ __forceinline__ void consume_gemv_mma(Ring& rg, const MegaArgs& A, const MegaGemv& g_mem, const MegaLayer* ly, int ctid,
                                             uint8_t* s_b, float* s_lnstat, float* s_mpart, float* s_xown, int* s_tr,
                                             const MmaGeom* s_geom, uint32_t xbar, unsigned& x_count) {
  using SM = MmaSmem<NR>;
  constexpr int NS = SM::NS;
  const MegaGemv g = g_mem;
  const MmaGeom mg = s_geom[g.shape];
  if (mg.rows_pad == 0) return;  // (CTA-uniform) more CTAs than octets: nothing to stream, nothing to compute
  const int lane = ctid & 31, warp = ctid >> 5;
  const int R = A.R;
  const int kblocks = g.K / 64;
  const bool ln = g.ln_s2 != nullptr;
  const int G = static_cast<int>(gridDim.x);
  // ---- activations: the fp16 exchange image IS the B operand -- one bulk copy; LayerNorm inputs bring the per-CTA shares
  //      of the row statistics along; both were issued by the thread that saw the preceding grid barrier open
  trace_ev(A, ctid, s_tr, 1);
  // ---- everything that does not need the activations happens while they travel: epilogue operands of this thread's
  //      outputs (bias, LayerNorm fold term, next LayerNorm's gain) and the lane's fragment addresses
  constexpr int NSLOT = (NR * MM_GROUP_ROWS + MG_CONS - 1) / MG_CONS;
  const int n_groups = mg.n_full + (mg.tail ? 1 : 0);
  const int first_rows = mg.n_full > 0 ? MM_GROUP_ROWS : mg.tail;
  const int wsh = (n_groups == 1 && first_rows <= 16) ? 4 : 6;  // outputs of a row per 16 / 64 consecutive threads
  float e_bias[NSLOT], e_s2[NSLOT], e_gain[NSLOT];
  auto prefetch_epi = [&](int gi, int rows) {
#pragma unroll
    for (int j = 0; j < NSLOT; ++j) {
      const int idx = ctid + j * MG_CONS;
      const int m = idx & ((1 << wsh) - 1), n = mg.lo + gi * MM_GROUP_ROWS + m;
      const bool ok = (idx >> wsh) < R && m < rows && n < mg.hi;
      e_bias[j] = (ok && g.bias != nullptr) ? __ldg(g.bias + n) : 0.f;
      e_s2[j] = (ok && ln) ? __ldg(g.ln_s2 + n) : 0.f;
      e_gain[j] = (ok && g.next_g != nullptr) ? __ldg(g.next_g + n) : 0.f;
    }
  };
  prefetch_epi(0, first_rows);
  const int gq = lane >> 2, tq = lane & 3;
  const int brow = gq < R ? gq : R - 1;  // lanes whose activation row does not exist read the last row: their output columns are never stored
  const uint32_t b_lane = smem_u32(s_b) + (brow * 4 + tq) * 16, b_plane = static_cast<uint32_t>(R * 64);
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8;
  uint32_t sw[4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) sw[ks] = ((2 * ks + (lane >> 4)) ^ (a_row & 7)) << 4;
  const uint32_t a_lane = rg.data0 + a_row * 128;
  unsigned unit = rg.unit;
  unsigned st = unit % NS, par = (unit / NS) & 1u;
  mbar_wait(xbar, x_count & 1u);
  ++x_count;
  trace_ev(A, ctid, s_tr, 2);
  for (int gi = 0; gi < n_groups; ++gi) {
    const bool full = gi < mg.n_full;
    const int rows = full ? MM_GROUP_ROWS : mg.tail;
    const int n_mt = (rows + 15) >> 4;
    const int units = full ? mg.units_full : mg.units_tail, kbu = full ? mg.kbu_full : mg.kbu_tail;
    if (gi > 0) prefetch_epi(gi, rows);
    float acc[4][4];
#pragma unroll
    for (int m = 0; m < 4; ++m)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[m][i] = 0.f;
    // main loop: warp w takes the k-blocks kb = w (mod 7) of every ring unit
    int kb_next = warp;  // this warp's next k-block of the group
    for (int u = 0, kb0 = 0; u < units; ++u, kb0 += kbu) {
      const int nkb = min(kbu, kblocks - kb0);
      // every warp waits for the unit (also the ones without a k-block in it: their arrival below must not run ahead of the ring)
      mbar_wait(rg.full(st), par);
      if (u == 0 && gi == 0) trace_ev(A, ctid, s_tr, 3);
      const int kbi = kb_next - kb0;
      const int n_it = kbi < nkb ? (nkb - kbi + MG_CONS_WARPS - 1) / MG_CONS_WARPS : 0;
      const uint32_t a_kb = a_lane + st * MG_STAGE_BYTES + kbi * rows * 128;
      const uint32_t b_kb = b_lane + kb_next * R * 128;
      const uint32_t a_step = MG_CONS_WARPS * rows * 128, b_step = MG_CONS_WARPS * R * 128;
      switch (n_mt) {
        case 1: mma_unit<1>(acc, a_kb, a_step, b_kb, b_step, n_it, sw, b_plane); break;
        case 2: mma_unit<2>(acc, a_kb, a_step, b_kb, b_step, n_it, sw, b_plane); break;
        case 3: mma_unit<3>(acc, a_kb, a_step, b_kb, b_step, n_it, sw, b_plane); break;
        default: mma_unit<4>(acc, a_kb, a_step, b_kb, b_step, n_it, sw, b_plane); break;
      }
      kb_next += n_it * MG_CONS_WARPS;
      __syncwarp();
      if (lane == 0) mbar_arrive(rg.empty(st));
      ++unit;
      if (++st == NS) {
        st = 0;
        par ^= 1u;
      }
    }
    trace_ev(A, ctid, s_tr, 4);
    // ---- row statistics (first group only): quantity q = (row, sum | sum of squares) is added up over the G per-CTA
    //      shares by 16 lanes, in a fixed order
    if (gi == 0 && ln) {
      const float* stp = reinterpret_cast<const float*>(s_b + SM::STAT_OFF);
      const int l = ctid & 15;
      const unsigned hmask = 0xFFFFu << (ctid & 16);  // the two 16-lane groups of a warp may run different trip counts
      for (int q = ctid >> 4; q < 2 * R; q += MG_CONS / 16) {  // (8 rows: 16 quantities, 14 lane groups)
        float t = 0.f;
        for (int i = l; i < G; i += 16) t += stp[i * 2 * R + q];
#pragma unroll
        for (int off = 8; off >= 1; off >>= 1) t += __shfl_xor_sync(hmask, t, off);
        if (l == 0) s_lnstat[q] = t;
      }
    }
    // ---- the warps' partial tiles -> shared memory [warp][activation row][weight row], summed by the epilogue threads
#pragma unroll
    for (int m = 0; m < 4; ++m)
      if (m < n_mt) {
        float* p = s_mpart + (warp * 8 + 2 * tq) * MM_PART_LD + m * 16 + gq;
        p[0] = acc[m][0];
        p[MM_PART_LD] = acc[m][1];
        p[8] = acc[m][2];
        p[MM_PART_LD + 8] = acc[m][3];
      }
    cons_sync();
    trace_ev(A, ctid, s_tr, 5);
#pragma unroll
    for (int j = 0; j < NSLOT; ++j) {
      const int idx = ctid + j * MG_CONS;
      const int r = idx >> wsh, m = idx & ((1 << wsh) - 1);
      const int n = mg.lo + gi * MM_GROUP_ROWS + m;
      const bool valid = r < R && m < rows && n < mg.hi;
      float v = 0.f;
      if (valid) {
#pragma unroll
        for (int w = 0; w < MG_CONS_WARPS; ++w) v += s_mpart[(w * 8 + r) * MM_PART_LD + m];
        if (ln) {
          const float mean = s_lnstat[2 * r] / g.K;
          const float rstd = rsqrtf(fmaxf(s_lnstat[2 * r + 1] / g.K - mean * mean, 0.f) + 1e-5f);
          v = rstd * (v - mean * e_s2[j]);
        }
        v += e_bias[j];
      }
      if (g.epi == GV_RESID) {  // (CTA-uniform; rows <= 16, one row per 16 lanes)
        float nv = 0.f;
        if (valid) {
          nv = s_xown[r * 16 + (n - mg.lo)] + v;
          s_xown[r * 16 + (n - mg.lo)] = nv;
        }
        if (j == 0 || (idx >> 5) * 32 < R * 16) publish_resid(A, r, n, valid, nv, e_gain[j], lane);  // (warp-uniform)
      } else if (valid) {
        switch (g.epi) {
          case GV_STORE:
            if (g.out16 != nullptr) g.out16[(static_cast<long long>(n >> 6) * R + r) * HEAD_DIM + (n & 63)] = __float2half_rn(v * 0.125f);  // cross-attention query [head][row][64], pre-scaled
            else g.out[static_cast<long long>(r) * g.ldo + n] = v;
            break;
          case GV_GELU:
            g.out16[act16_off(R, r, n)] = __float2half_rn(gelu_erf(v));
            break;
          case GV_QKV: {
            const int d = A.d;
            if (n < d) {  // self-attention query [head][row][64], pre-scaled
              A.q16[(static_cast<long long>(n >> 6) * R + r) * HEAD_DIM + (n & 63)] = __float2half_rn(v * 0.125f);
            } else {
              const int pos = row_pos(A, r);
              __half* cache = (n < 2 * d) ? ly->kcache : ly->vcache;
              const int e = (n < 2 * d) ? n - d : n - 2 * d;
              cache[(static_cast<long long>(row_slot(A, r)) * A.t_max + pos) * d + e] = __float2half_rn(v);
            }
            break;
          }
          default:
            break;
        }
      }
    }
    if (gi + 1 < n_groups) cons_sync();  // the partial tiles are rewritten by the next group
  }
  trace_ev(A, ctid, s_tr, 6);
  rg.unit = unit;
}

// ------------------------------------------------------------------ warp-MMA pass: cross-query GEMV fused into the cross-attention
// A grid-wide phase has a fixed latency (release fence, counter, poll, reload) whatever it computes, so the
// LayerNorm + cross-query projection no longer has one: every key-split CTA of head h computes the head's 64 query columns
// itself (all R rows: 64 x 1280 weights = 164 KB per CTA through the ring, the same bytes for the 7 splits of a head, so HBM
// still reads W once and the L2 serves the rest), then walks its keys as before.  Weight image: mega_mma_image with one
// "owner" per head.  B operand (the LayerNorm-scaled residual rows) and statistic shares: reloaded by the barrier's opener.
template <int NS>
__device__ __forceinline__ void produce_cross_fused(Ring& rg, const MegaArgs& A, const MegaLayer& ly, const MmaGeom* s_geom) {
  const CrossGeom cg = cross_geom(A.n_utt, A.H);
  const uint64_t pol = l2_policy_evict_first();
  const int kblocks = A.d / 64, units = s_geom[4].units_full, kbu = s_geom[4].kbu_full;  // 64-row group, K = d
  for (int task = blockIdx.x; task < cg.n_tasks; task += gridDim.x) {
    const int split = task % cg.S, uh = task / cg.S;
    const int h = uh % A.H;
    const __half* wq = ly.cq.w + static_cast<long long>(h) * 64 * A.d;
    for (int u = 0; u < units; ++u) {
      const int kb0 = u * kbu, nkb = min(kbu, kblocks - kb0);
      const int st = rg.unit % NS;
      mbar_wait(rg.empty(st), ((rg.unit / NS) & 1u) ^ 1u);
      mbar_arrive_expect_tx(rg.full(st), static_cast<uint32_t>(nkb * 64 * 128));
      bulk_load_1d_hint(rg.data0 + st * MG_STAGE_BYTES, wq + static_cast<long long>(kb0) * 64 * 64, static_cast<uint32_t>(nkb * 64 * 128),
                        rg.full(st), pol);
      ++rg.unit;
    }
    const int t0 = split * cg.KS;
    const int nk = max(0, min(cg.KS, T_ENC_PAD - t0));  // (splits past the last row: see produce_cross_impl)
    const long long off = (static_cast<long long>(uh) * T_ENC_PAD + t0) * HEAD_DIM;
    for (int kv = 0; kv < 2; ++kv) {
      const int st = rg.unit % NS;
      mbar_wait(rg.empty(st), ((rg.unit / NS) & 1u) ^ 1u);
      mbar_arrive_expect_tx(rg.full(st), static_cast<uint32_t>(nk * HEAD_DIM * 2));
      if (nk > 0)
        bulk_load_1d_hint(rg.data0 + st * MG_STAGE_BYTES, (kv == 0 ? ly.ck : ly.cv) + off, static_cast<uint32_t>(nk * HEAD_DIM * 2),
                          rg.full(st), pol);
      ++rg.unit;
    }
  }
}

template <int NB, int NS>
__device__ __forceinline__ void consume_cross_fused(Ring& rg, const MegaArgs& A, const MegaLayer& ly, int ctid, uint8_t* s_b, float* s_mpart,
                                                    float* s_lnstat, int* s_tr, const MmaGeom* s_geom, uint32_t xbar, unsigned& x_count,
                                                    unsigned tag, int stat_off) {
  float* s_part = reinterpret_cast<float*>(s_b);  // attention scratch: merge area, queries at +4096 floats
  float* s_q = s_part + 4096;
  const MegaGemv g = ly.cq;
  const int lane = ctid & 31, warp = ctid >> 5, gq = lane >> 2, tq = lane & 3;
  const int R = A.R, d = A.d, beam = A.beam, H = A.H, G = static_cast<int>(gridDim.x);
  const CrossGeom cg = cross_geom(A.n_utt, H);
  const int kblocks = d / 64, units = s_geom[4].units_full, kbu = s_geom[4].kbu_full;
  const uint32_t ring_data0 = rg.data0, ring_full0 = rg.full0, ring_empty0 = rg.empty0;
  unsigned unit = rg.unit;
  trace_ev(A, ctid, s_tr, 10);
  // the LayerNorm-scaled residual rows + statistic shares (issued by the thread that saw the barrier open)
  mbar_wait(xbar, x_count & 1u);
  ++x_count;
  {  // row statistics, as in consume_gemv_mma
    const float* stp = reinterpret_cast<const float*>(s_b + stat_off);
    const int l = ctid & 15;
    const unsigned hmask = 0xFFFFu << (ctid & 16);
    for (int q = ctid >> 4; q < 2 * R; q += MG_CONS / 16) {
      float t = 0.f;
      for (int i = l; i < G; i += 16) t += stp[i * 2 * R + q];
#pragma unroll
      for (int off = 8; off >= 1; off >>= 1) t += __shfl_xor_sync(hmask, t, off);
      if (l == 0) s_lnstat[q] = t;
    }
  }
  const int brow = gq < R ? gq : R - 1;
  const uint32_t b_lane = smem_u32(s_b) + FUSED_B_OFF + (brow * 4 + tq) * 16, b_plane = static_cast<uint32_t>(R * 64);
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8;
  uint32_t sw[4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) sw[ks] = ((2 * ks + (lane >> 4)) ^ (a_row & 7)) << 4;
  const uint32_t a_lane = ring_data0 + a_row * 128;
  constexpr int NSLOT = (NB * 64 + MG_CONS - 1) / MG_CONS;
  for (int task = blockIdx.x; task < cg.n_tasks; task += gridDim.x) {
    const int split = task % cg.S, uh = task / cg.S;
    const int u = uh / H, h = uh - u * H;
    const int t0 = split * cg.KS;
    int nk = min(cg.KS, T_ENC - t0);  // keys >= 1500 (padding rows) are never touched
    if (nk < 0) nk = 0;
    // ---- cross-query projection of head h: 64 weight rows x all R rows
    float e_bias[NSLOT], e_s2[NSLOT];
#pragma unroll
    for (int j = 0; j < NSLOT; ++j) {
      const int idx = ctid + j * MG_CONS;
      const bool ok = (idx >> 6) < R;
      e_bias[j] = ok ? __ldg(g.bias + h * 64 + (idx & 63)) : 0.f;
      e_s2[j] = ok ? __ldg(g.ln_s2 + h * 64 + (idx & 63)) : 0.f;
    }
    float acc[4][4];
#pragma unroll
    for (int m = 0; m < 4; ++m)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[m][i] = 0.f;
    int kb_next = warp;
    for (int uu = 0, kb0 = 0; uu < units; ++uu, kb0 += kbu, ++unit) {
      const int nkb = min(kbu, kblocks - kb0);
      const unsigned st = unit % NS;
      mbar_wait(ring_full0 + 8u * st, (unit / NS) & 1u);
      const int kbi = kb_next - kb0;
      const int n_it = kbi < nkb ? (nkb - kbi + MG_CONS_WARPS - 1) / MG_CONS_WARPS : 0;
      mma_unit<4>(acc, a_lane + st * MG_STAGE_BYTES + kbi * 64 * 128, MG_CONS_WARPS * 64 * 128, b_lane + kb_next * R * 128,
                  MG_CONS_WARPS * R * 128, n_it, sw, b_plane);
      kb_next += n_it * MG_CONS_WARPS;
      __syncwarp();
      if (lane == 0) mbar_arrive(ring_empty0 + 8u * st);
    }
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      float* p = s_mpart + (warp * 8 + 2 * tq) * MM_PART_LD + m * 16 + gq;
      p[0] = acc[m][0];
      p[MM_PART_LD] = acc[m][1];
      p[8] = acc[m][2];
      p[MM_PART_LD + 8] = acc[m][3];
    }
    cons_sync();
#pragma unroll
    for (int j = 0; j < NSLOT; ++j) {
      const int idx = ctid + j * MG_CONS;
      const int r = idx >> 6, c = idx & 63;
      const int rl = r - u * beam;  // row inside the utterance
      if (r < R && rl >= 0 && rl < beam) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < MG_CONS_WARPS; ++w) v += s_mpart[(w * 8 + r) * MM_PART_LD + c];
        const float mean = s_lnstat[2 * r] / d;
        const float rstd = rsqrtf(fmaxf(s_lnstat[2 * r + 1] / d - mean * mean, 0.f) + 1e-5f);
        v = rstd * (v - mean * e_s2[j]) + e_bias[j];
        reinterpret_cast<__half*>(s_q)[rl * 72 + c] = __float2half_rn(v * 0.125f);  // pre-scaled query; 144-byte rows: conflict-free fragment loads
      }
    }
    cons_sync();
    trace_ev(A, ctid, s_tr, 11);
    // ---- warp-MMA walk (FlashAttention-2 register layout): S = Q K^T with the utterance's <= 8 beams as the MMA's M rows
    //      (rows 8..15 are zero), 16 keys per block, 7 warps over the blocks; P stays in registers as the A operand of
    //      O += P V (V through ldmatrix.trans).  Every warp ends with (m, l, O[64]) per beam, merged in cross_tail.
    const int stK = unit % NS, stV = (unit + 1) % NS;
    uint32_t aq[4][2];
    {
      const bool row_ok = gq < beam;
      const uint32_t qa = smem_u32(s_q) + (row_ok ? gq : 0) * 144 + tq * 4;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        aq[ks][0] = row_ok ? lds32(qa + ks * 32) : 0u;
        aq[ks][1] = row_ok ? lds32(qa + ks * 32 + 16) : 0u;
      }
    }
    float m_run = -INFINITY, l_run = 0.f;
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) o[j][i] = 0.f;
    mbar_wait(ring_full0 + 8u * stK, (unit / NS) & 1u);
    mbar_wait(ring_full0 + 8u * stV, ((unit + 1) / NS) & 1u);
    trace_ev(A, ctid, s_tr, 12);
    // (the cross K/V rows arrive chunk-swizzled by the key index -- gemm_tc.cu EPI_CROSSKV kv_swizzle -- so ldmatrix is
    //  conflict-free: lane's row inside a 16-key half, 16-byte chunk (2 kq + lane / 16) ^ (key & 7))
    const uint32_t lane_row = static_cast<uint32_t>(((lane & 7) + ((lane >> 3) & 1) * 8) * 128);
    const uint32_t lane_c = static_cast<uint32_t>(lane >> 4), lane_x = static_cast<uint32_t>(lane & 7);
    const uint32_t sKl = ring_data0 + stK * MG_STAGE_BYTES + lane_row, sVl = ring_data0 + stV * MG_STAGE_BYTES + lane_row;
    for (int blk = warp; blk * 32 < nk; blk += MG_CONS_WARPS) {  // 32 keys per trip: 4 score tiles of 8 keys
      float sc[4][4];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) sc[nt][i] = 0.f;
#pragma unroll
      for (int kq = 0; kq < 4; ++kq) {
        const uint32_t a4[4] = {aq[kq][0], 0u, aq[kq][1], 0u};
#pragma unroll
        for (int half = 0; half < 2; ++half) {  // keys 16 half .. 16 half + 15 of the block
          uint32_t kf[4];
          ldmatrix_x4(sKl + blk * 4096 + half * 2048 + (((2 * kq + lane_c) ^ lane_x) << 4), kf);
          mma_m16n8k16(sc[2 * half], a4, kf[0], kf[2]);
          mma_m16n8k16(sc[2 * half + 1], a4, kf[1], kf[3]);
        }
      }
      // online softmax of row gq over the block's 32 keys (keys 8 nt + 2 tq, + 1 live in this lane)
      float sv[8];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int k0 = blk * 32 + nt * 8 + 2 * tq;
        sv[2 * nt] = k0 < nk ? sc[nt][0] : -INFINITY;
        sv[2 * nt + 1] = k0 + 1 < nk ? sc[nt][1] : -INFINITY;
      }
      float mx = sv[0];
#pragma unroll
      for (int q = 1; q < 8; ++q) mx = fmaxf(mx, sv[q]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m_run, mx);
      const float al = __expf(m_run - mn);
      float pr[8], rs = 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        pr[q] = __expf(sv[q] - mn);
        rs += pr[q];
      }
      rs += __shfl_xor_sync(0xffffffffu, rs, 1);
      rs += __shfl_xor_sync(0xffffffffu, rs, 2);
      l_run = fmaf(l_run, al, rs);
      m_run = mn;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j][0] *= al;
        o[j][1] *= al;
      }
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {  // 16 keys per k-step
        __half2 h01 = __floats2half2_rn(pr[4 * kk], pr[4 * kk + 1]), h23 = __floats2half2_rn(pr[4 * kk + 2], pr[4 * kk + 3]);
        const uint32_t pa[4] = {*reinterpret_cast<uint32_t*>(&h01), 0u, *reinterpret_cast<uint32_t*>(&h23), 0u};
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {
          uint32_t vf[4];
          ldmatrix_x4_trans(sVl + blk * 4096 + kk * 2048 + (((2 * jp + lane_c) ^ lane_x) << 4), vf);
          mma_m16n8k16(o[2 * jp], pa, vf[0], vf[1]);
          mma_m16n8k16(o[2 * jp + 1], pa, vf[2], vf[3]);
        }
      }
    }
    trace_ev(A, ctid, s_tr, 13);
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(ring_empty0 + 8u * stK);
      mbar_arrive(ring_empty0 + 8u * stV);
    }
    unit += 2;
    if (gq < beam) {
      float* dst = s_part + (warp * NB + gq) * 66;
#pragma unroll
      for (int j = 0; j < 8; ++j) *reinterpret_cast<float2*>(dst + 8 * j + 2 * tq) = make_float2(o[j][0], o[j][1]);
      if (tq == 0) {
        dst[64] = m_run;
        dst[65] = l_run;
      }
    }
    cross_tail<NB, false, true>(A, cg, ctid, s_part, tag, s_tr, xbar, &x_count, uh, u, h, split, beam, ring_empty0, stK, stV);
  }
  rg.unit = unit;
}

template <int NR>
__global__ void __launch_bounds__(MG_THREADS, 1) dec_pass_mma_kernel(const MegaArgs A) {
  if (A.pf_len == 0 && A.st->all_done) return;  // a step enqueued ahead of the host's poll (every thread of every CTA leaves)
  using SM = MmaSmem<NR>;
  constexpr int NS = SM::NS;
  extern __shared__ __align__(1024) uint8_t mg_smem[];
  uint8_t* s_b = mg_smem + SM::OFF_B;
  float* s_part = reinterpret_cast<float*>(s_b);  // attention scratch: the attention phases never touch the B operand
  float* s_mpart = reinterpret_cast<float*>(mg_smem + SM::OFF_PART);
  uint64_t* bars = reinterpret_cast<uint64_t*>(mg_smem + SM::OFF_BARS);
  float* s_stat = reinterpret_cast<float*>(mg_smem + SM::OFF_STAT);
  float* s_lnstat = s_stat;  // [0, 16): row statistics of the current LayerNorm phase
  unsigned short* s_slot_tab = reinterpret_cast<unsigned short*>(mg_smem + SM::OFF_SLOT);
  MegaLayer* s_ly = reinterpret_cast<MegaLayer*>(mg_smem + SM::OFF_LY);
  MmaGeom* s_geom = reinterpret_cast<MmaGeom*>(mg_smem + SM::OFF_GEOM);
  float* s_xown = s_stat + 784;
  int* s_tr = reinterpret_cast<int*>(s_stat + 16);  // [16, 784): event trace (1 + 2 x 380 words)
  Ring rg;
  rg.data = mg_smem;
  rg.data0 = smem_u32(mg_smem);
  rg.full0 = smem_u32(bars);
  rg.empty0 = rg.full0 + 8 * NS;
  rg.unit = 0;
  const uint32_t xbar = rg.full0 + 8 * (2 * NS);  // activation reload (bulk copy) of the GEMV phases
  unsigned x_count = 0;
  const int tid = threadIdx.x;
  if ((smem_u32(mg_smem) & 1023u) != 0) __trap();  // the swizzled weight boxes need 1024-byte alignment
  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(rg.full(s), 1);
      mbar_init(rg.empty(s), MG_CONS_WARPS);
    }
    mbar_init(xbar, 1);
    fence_mbar_init();
  }
  if (tid < 5) {  // geometry of the five GEMV shapes (MegaGemv::shape)
    const int d = A.d;
    const int Ns[5] = {3 * d, d, 4 * d, d, A.vocab.N}, Ks[5] = {d, d, d, 4 * d, d};
    s_geom[tid] = mma_geom(Ns[tid], Ks[tid]);
  }
  __syncthreads();
  const int L = A.n_layers;

  if (tid >= MG_CONS) {
    // ============================ producer: the static weight / KV stream of this CTA
    if (tid == MG_CONS) {
      // (one call site per function, everything inlined: a call would park the kernel arguments and the live registers in
      //  local memory, and every acquire of the barrier invalidates the L1 -- each access after it was an L2 round trip)
      for (int l = 0; l <= L; ++l) {
        if (l == L) {
          if (A.with_logits) produce_gemv_mma<NS>(rg, A.vocab, s_geom, A.dbg);
          break;
        }
        const MegaLayer& ly = A.layers[l];
        for (int j = 0; j < 6; ++j) {  // qkv, o, [cross-q of the task's head + cross K/V], cross-o, fc1, fc2
          if (j == 2) produce_cross_fused<NS>(rg, A, ly, s_geom);
          else produce_gemv_mma<NS>(rg, (&ly.qkv)[j], s_geom, A.dbg);  // (index 2, the cross-query GEMV, is the fused phase's)
        }
      }
    }
    return;
  }
  // ============================== consumers
  const int ctid = tid;
  unsigned epoch = *A.epoch_base;
  const unsigned epoch0 = epoch;
  if (ctid == 0) s_tr[0] = -1;
  if (A.trace != nullptr && blockIdx.x == 0 && ctid == 0) A.trace[0] = globaltimer_ns();
  auto prefetch_layer = [&](int l) {
    if (ctid < static_cast<int>(sizeof(MegaLayer) / 16))
      cp_async16(smem_u32(reinterpret_cast<uint8_t*>(s_ly) + (l & 1) * MG_LY_STRIDE) + ctid * 16,
                 reinterpret_cast<const uint8_t*>(A.layers + l) + ctid * 16);
  };
  if (L > 0) prefetch_layer(0);
  const int pos_dec = A.pf_len > 0 ? 0 : A.st->pos;
  const int flipv = *A.flip;
  if (A.pf_len == 0 && (ctid >> 5) < SA_WARPS) {
    const int task = (ctid >> 5) * static_cast<int>(gridDim.x) + static_cast<int>(blockIdx.x);  // consume_self_attn_mma's first task of this warp
    if (task < A.R * A.H) {
      const int* indir = (flipv ? A.indir1 : A.indir0) + static_cast<long long>(task / A.H) * A.t_max;
      for (int t = ctid & 31; t < pos_dec; t += 32) s_slot_tab[(ctid >> 5) * 448 + t] = static_cast<unsigned short>(indir[t]);
    }
  }
  cp_async_wait_all();
  {
    // token + positional embedding: every CTA produces (and keeps) the residual-stream columns it owns and publishes them
    // for layer 0's LayerNorm + QKV phase (16 lanes per row)
    const MmaGeom mg = s_geom[1];
    const float* gain0 = L > 0 ? A.layers[0].qkv.ln_g : A.vocab.ln_g;
    for (int base = 0; base < A.R * 16; base += MG_CONS) {
      const int idx = base + ctid;
      const int r = idx >> 4, c = idx & 15, n = mg.lo + c;
      const bool valid = r < A.R && n < mg.hi;
      float v = 0.f, gain = 0.f;
      if (valid) {
        v = __half2float(A.tok_emb[static_cast<long long>(row_token(A, r)) * A.d + n]) + A.pos_emb[static_cast<long long>(row_pos(A, r)) * A.d + n];
        gain = __ldg(gain0 + n);
        s_xown[r * 16 + c] = v;
      }
      if ((idx >> 5) * 32 < A.R * 16) publish_resid(A, r, n, valid, v, gain, ctid & 31);  // (warp-uniform)
    }
  }
  const uint32_t sba = smem_u32(s_b);
  // Phase loop with ONE inlined copy of every phase function and of the barrier (see the producer's note): layer l runs the
  // phases 0 qkv, 1 self-attention, 2 out-proj, 3 cross-attention (with its query projection), 4 cross-out, 5 fc1, 6 fc2;
  // "layer" L is the vocabulary projection alone.  The barrier that ends a phase issues the activation reload of the GEMV that follows.
  Reload rl_next = L > 0 ? gemv_reload(A, A.layers[0].qkv, s_geom) : (A.with_logits ? gemv_reload(A, A.vocab, s_geom) : Reload());
  for (int l = -1; l <= L; ++l) {
    const bool vocab_layer = l == L;
    if (vocab_layer && !A.with_logits) break;
    const MegaLayer& ly = *reinterpret_cast<const MegaLayer*>(reinterpret_cast<const uint8_t*>(s_ly) + ((l < 0 ? 0 : l) & 1) * MG_LY_STRIDE);
    if (l >= 0 && l + 1 < L) prefetch_layer(l + 1);
    if (l >= 0) trace_open(A, ctid, s_tr, l);
    const int n_ph = (l < 0 || vocab_layer) ? 1 : 7;
    for (int ph = 0; ph < n_ph; ++ph) {
      if (l < 0) {
        // (the embedding phase ran above; this iteration only lends its barrier)
      } else if (!vocab_layer && ph == 1) {
        consume_self_attn_mma(A, ly, ctid, reinterpret_cast<uint8_t*>(s_part), s_slot_tab, pos_dec, flipv, s_tr);
      } else if (!vocab_layer && ph == 3) {
        consume_cross_fused<NR, NS>(rg, A, ly, ctid, s_b, s_mpart, s_lnstat, s_tr, s_geom, xbar, x_count, epoch + 1, SM::STAT_OFF);
      } else {
        const MegaGemv& g = vocab_layer ? A.vocab : (&ly.qkv)[ph == 0 ? 0 : (ph == 2 ? 1 : ph - 1)];
        consume_gemv_mma<NR>(rg, A, g, &ly, ctid, s_b, s_lnstat, s_mpart, s_xown, s_tr, s_geom, xbar, x_count);
      }
      Reload rl = rl_next;
      if (l >= 0) {
        rl = Reload();
        if (!vocab_layer) {
          if (ph == 6) {
            cp_async_wait_all();  // the next layer's descriptor has landed; the barrier's CTA sync publishes it
            // (all layers share the GEMV shapes and the exchange buffers: this layer's qkv descriptor stands for the next one's)
            rl = l + 1 < L ? gemv_reload(A, ly.qkv, s_geom) : (A.with_logits ? gemv_reload(A, A.vocab, s_geom) : Reload());
          } else if (ph == 2) {  // next: cross-attention with its own query projection (B operand above the merge area)
            rl.src = ly.cq.x16;  // (every CTA: also the ones that own no column of a d-wide GEMV wait for it)
            rl.bytes = static_cast<uint32_t>((A.d / 64) * A.R * 128);
            rl.src2 = A.xstat;
            rl.bytes2 = static_cast<uint32_t>(gridDim.x * A.R * 8);
            rl.dst_off = FUSED_B_OFF;
          } else if (ph != 0) {  // 1 -> out-proj, 3 -> cross-out, 4 -> fc1, 5 -> fc2
            rl = gemv_reload(A, (&ly.qkv)[ph == 1 ? 1 : ph], s_geom);
          }
        }
      }
      grid_barrier_mma(A, epoch, ctid, epoch0, rl, sba, SM::STAT_OFF, xbar, s_tr);
    }
  }
  trace_dump(A, ctid, s_tr);
  if (blockIdx.x == 0 && ctid == 0) {
    *A.epoch_base = epoch;
    A.epoch_base[8] = epoch * gridDim.x;
  }
}

__global__ void chunk_major_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int N, int K, int n_chunks) {
  const int kc = K / n_chunks;
  const long long total = static_cast<long long>(N) * K / 8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long e = i * 8;
    const int n = static_cast<int>(e / K), k = static_cast<int>(e - static_cast<long long>(n) * K);
    const int c = k / kc, kk = k - c * kc;
    *reinterpret_cast<uint4*>(dst + (static_cast<long long>(c) * N + n) * kc + kk) = *reinterpret_cast<const uint4*>(src + e);
  }
}

// W [N][K] row-major -> the warp-MMA image: CTA b of a `G`-CTA pass owns the rows [lo_b, lo_b + rows_b) (N / G each, the first
// N % G CTAs one more); inside, groups of 64 rows, each stored [k-block][rows][64] with the 16-byte chunks of a row
// XOR-swizzled by (row & 7).  One ring unit = a contiguous run of k-blocks = ONE bulk copy, and the bytes land in
// shared memory exactly as ldmatrix wants them (one contiguous copy per unit instead of a TMA tensor-map load per
// k-block, so that a phase's weights are in place when its barrier opens).
__global__ void mma_image_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int N, int K, int G) {
  const int base = N / G, rem = N - base * G;
  const int big = rem * (base + 1);
  const int kc = K >> 3;
  const long long total = static_cast<long long>(N) * kc;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(i / kc), c16 = static_cast<int>(i - static_cast<long long>(n) * kc);
    int lo, rows;
    if (n < big) {
      rows = base + 1;
      lo = (n / rows) * rows;
    } else {
      rows = base;
      lo = big + ((n - big) / rows) * rows;
    }
    const int rl = n - lo, gi = rl >> 6, row = rl & 63;
    const int rows_g = min(64, rows - gi * 64);
    const int kb = c16 >> 3, c = c16 & 7;
    const uint4 v = *reinterpret_cast<const uint4*>(src + static_cast<long long>(n) * K + c16 * 8);
    *reinterpret_cast<uint4*>(dst + static_cast<long long>(lo + gi * 64) * K + static_cast<long long>(kb) * rows_g * 64 + row * 64 + ((c ^ (row & 7)) << 3)) = v;
  }
}

}  // namespace

void mega_mma_image(const __half* src, __half* dst, int N, int K, int grid, cudaStream_t stream) {
  mma_image_kernel<<<1024, 256, 0, stream>>>(src, dst, N, K, grid);
  WISB_CUDA(cudaGetLastError());
}

__global__ void ln_fold_kernel(const __half* __restrict__ w, const float* __restrict__ g, const float* __restrict__ b,
                               const float* __restrict__ bias, float* __restrict__ s2, float* __restrict__ biasf, int N, int K) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  float a = 0.f, c = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float wv = __half2float(w[static_cast<long long>(n) * K + k]);
    a = fmaf(g[k], wv, a);
    c = fmaf(b[k], wv, c);
  }
  a = warp_sum(a);
  c = warp_sum(c);
  if (lane == 0) {
    s2[n] = a;
    biasf[n] = c + (bias != nullptr ? bias[n] : 0.f);
  }
}

void mega_ln_fold(const __half* w, const float* g, const float* b, const float* bias, float* s2, float* biasf, int N, int K,
                  cudaStream_t stream) {
  ln_fold_kernel<<<cdiv(N, 8), 256, 0, stream>>>(w, g, b, bias, s2, biasf, N, K);
  WISB_CUDA(cudaGetLastError());
}

int mega_k_chunks(int K) {
  int n = (K + MG_KC_MAX - 1) / MG_KC_MAX;
  while (K % (8 * n) != 0) ++n;
  return n;
}

// W [N][K] -> [chunk][N][K / n_chunks]: every (chunk, row range) the pass kernel streams becomes one contiguous block
void mega_chunk_major(const __half* src, __half* dst, int N, int K, cudaStream_t stream) {
  chunk_major_kernel<<<1024, 256, 0, stream>>>(src, dst, N, K, mega_k_chunks(K));
  WISB_CUDA(cudaGetLastError());
}

size_t mega_flags_words() { return 160 * 32 + 32; }

void dec_pass_run(const MegaArgs& a, int num_sms, cudaStream_t stream) {
  WISB_REQUIRE(a.R >= 1 && a.R <= 8, "decoder pass: 1..8 rows");
  WISB_REQUIRE(a.d % 64 == 0 && a.d <= MG_KC_MAX, "decoder pass: d_model <= 1536");
  WISB_REQUIRE((a.d + num_sms - 1) / num_sms <= 16, "decoder pass: too few SMs for the per-CTA residual slice");
  WISB_REQUIRE(num_sms <= 160, "decoder pass: more SMs than barrier flags");
  static std::atomic<unsigned long long> once{0};  // per device: function attributes belong to the device's context
  once_per_device(once, [] {
    WISB_CUDA(cudaFuncSetAttribute(dec_pass_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, MG_SMEM));
    WISB_CUDA(cudaFuncSetAttribute(dec_pass_kernel<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, MG_SMEM));
    WISB_CUDA(cudaFuncSetAttribute(dec_pass_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, MG_SMEM));
  });
  void* args[] = {const_cast<MegaArgs*>(&a)};
  if (a.tc) {
    static std::atomic<unsigned long long> once_mma{0};
    once_per_device(once_mma, [] {
      WISB_CUDA(cudaFuncSetAttribute(dec_pass_mma_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, MmaSmem<2>::TOTAL));
      WISB_CUDA(cudaFuncSetAttribute(dec_pass_mma_kernel<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, MmaSmem<5>::TOTAL));
      WISB_CUDA(cudaFuncSetAttribute(dec_pass_mma_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, MmaSmem<8>::TOTAL));
    });
    WISB_REQUIRE(a.d % 64 == 0 && 4 * a.d <= 5120, "warp-MMA decoder pass: d_model <= 1280");
    WISB_REQUIRE((a.d + num_sms - 1) / num_sms <= 16, "warp-MMA decoder pass: too few SMs for the per-CTA residual slice");
    if (a.R <= 2) {
      WISB_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(dec_pass_mma_kernel<2>), dim3(num_sms), dim3(MG_THREADS), args, MmaSmem<2>::TOTAL, stream));
    } else if (a.R <= 5) {
      WISB_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(dec_pass_mma_kernel<5>), dim3(num_sms), dim3(MG_THREADS), args, MmaSmem<5>::TOTAL, stream));
    } else {
      WISB_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(dec_pass_mma_kernel<8>), dim3(num_sms), dim3(MG_THREADS), args, MmaSmem<8>::TOTAL, stream));
    }
    return;
  }
  const void* fn = a.R <= 2 ? reinterpret_cast<const void*>(dec_pass_kernel<2>)
                            : a.R <= 5 ? reinterpret_cast<const void*>(dec_pass_kernel<5>)
                                       : reinterpret_cast<const void*>(dec_pass_kernel<8>);
  WISB_CUDA(cudaLaunchCooperativeKernel(fn, dim3(num_sms), dim3(MG_THREADS), args, MG_SMEM, stream));
}

}  // namespace wisb
