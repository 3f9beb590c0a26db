// Device-side token search: logits processors, log-softmax, top-k over beam x vocabulary and the CTranslate2-style
// beam / greedy bookkeeping, all without a host round trip (the host only polls DecState::all_done).
//
// Semantics restated from CTranslate2 4.1.0 as listed in SURVEY.md section 8a rows A11-A13 (the reference call is
// main.py:687-692 with the library defaults patience=1, length_penalty=1, suppress_blank=True,
// suppress_tokens=[-1], num_hypotheses=1):
//   * processors: `suppress_ids` -> -inf every step; {blank, eot} -> -inf at the first generated step
//   * scores: log_softmax(logits) + cumulative beam score, divided by (step+1)^length_penalty
//   * candidates: top 2*beam of beam*V (ties: lowest flat index); at step 0 only beam 0 is live
//   * the first `beam` candidates that end in eot (or any at the last step) become hypotheses and are replaced by the
//     next non-eot candidates; an utterance is finished once round(beam*patience) hypotheses exist or at the last step
//     (a cap of 0 new tokens: at once, with no hypothesis); a row left without a candidate is dead (eot, cum -inf)
//   * result: best normalised score, first one on ties; eot itself is not part of the output
//   * beam_size == 1 is the same procedure with 2 candidates, i.e. greedy arg-max decoding
// Timestamp mode (SearchArgs::ts, prompt without <|notimestamps|>) adds Whisper's timestamp rules after those processors
// (openai/whisper, transformers' WhisperTimeStampLogitsProcessor): <|notimestamps|> off; at the first step text off and
// timestamps above ts_max_init off; after a timestamp pair timestamps off, after a lone timestamp text (< eot) off;
// timestamps below the last one off (at or below it unless it opened a pair); and text off in a row whose timestamp
// log-sum-exp exceeds its best text logit.  The vocabulary is then split as 32 text chunks + one timestamp chunk.
//
// History processors (SearchArgs::rep_penalty != 1 or no_repeat_ngram > 0; CTranslate2's repetition_penalty and
// no_repeat_ngram_size).  hist = the row's generated tokens seq[*flip][r][0, gen), after beam reordering: timestamp
// tokens count, prompt tokens do not.  Pinned to transformers' RepetitionPenaltyLogitsProcessor and
// NoRepeatNGramLogitsProcessor with input_ids = hist (tests/golden/history_processors_hf.npz); CTranslate2's own
// implementation is UNPINNED (it probably also counts the last prompt token, from which its search starts).
//   * repetition_penalty p: every distinct id in hist gets l < 0 ? l * p : l / p, once however often it occurs
//   * no_repeat_ngram_size n: if gen + 1 >= n, every hist[i + n - 1] with hist[i .. i + n - 2] == hist[gen - n + 1 ..
//     gen - 1], 0 <= i <= gen - n, is -inf (n = 1: every id in hist)
//   * order: penalty on the raw logits, n-gram ban, the suppress masks, then the timestamp rules (rule 5 sees the
//     penalised logits), then log-softmax and top-k as above.  Each processor is one fp32 IEEE operation, so the result
//     is bit-exact; an id the masks turn off is -inf whatever the processors did.
// They run in the topk_partial_kernel<NCH, true> instantiation, picked only when one is on: each (chunk, row) block
// stages hist in shared memory and flags its chunk's ids before it reads the logits.
// Per-utterance beam, patience and length penalty (SearchArgs::beam_u; a call that mixes windows with different search
// options): every utterance keeps a block of `beam` rows (the call's largest beam B) and searches only its first b_u
// rows, with 2 b_u candidates, its own max_hyp and length penalty; rows b_u .. B - 1 are dead from search_init on (eot,
// cum -inf) and never become a candidate or a hypothesis.  topk_partial_kernel is shared: it still emits 2 B partials
// per chunk, of which the merge takes the first 2 b_u (a chunk's partials are sorted, so this is the chunk's top 2 b_u).
// Only the search_tail_kernel<NCH, true> / search_init_kernel<true> instantiations read the per-utterance arrays; a call
// whose windows agree runs the <false> ones.
//
// Sampling (SearchArgs::sample: beam_size 1 and sampling_topk != 1; CTranslate2's RandomSampler with num_hypotheses n,
// made deterministic by a per-window seed).  Each window keeps a block of n = `beam` rows, one per hypothesis; rows are
// independent and never reorder (indir[r][pos] = r, a row's history is its own) and every row is live at gen 0.  One
// step of row r of window u, hypothesis k = r mod n, generated-token index gen:
//   1. the processors above run unchanged (penalty, n-gram ban, masks, timestamp rules including rule 5), giving the
//      processed logits l_v and the row's lse over them;
//   2. candidates S: topk == 0 every v with a finite l_v; topk == K in [2, 16] the K largest finite l_v (ties: lowest
//      id); rule 5 (ts_only) keeps only the timestamps, as for beam rows;
//   3. noise: x = word 0 of Philox4x32-10 with counter (v, gen, k, 0) and key (lo32(seed_u), hi32(seed_u));
//      u = ((x >> 9) + 0.5) * 2^-23 (exact in fp32, in (0, 1)); g_v = -logf(-logf(u)) in fp32;
//   4. sample: the v in S with the largest key_v = fp32(l_v / T) + g_v (IEEE division), ties to the lowest id.  This is
//      Gumbel-max: v ~ softmax(l_S / T), transformers' TemperatureLogitsWarper followed by TopKLogitsWarper;
//   5. cum += l_v - lse, the untempered log-prob (CTranslate2's RandomSampler gathers from the untempered scores;
//      UNPINNED like the rest of its search).
// A row finishes when it samples eot or at its window's last step; its hypothesis is its tokens without eot, scored
// cum / (gen + 1)^length_penalty in fp32 (beam 1's normalisation), and it is dead from then on (eot, cum -inf).  A row
// left with an empty S is dead with no hypothesis (empty, score -inf).  A window is done once all its rows are.
// topk == 0 runs topk_partial_kernel<NCH, HIST, true>: each (chunk, row) block draws the noise of its finite tokens and
// emits the chunk's best packed (key, id) in part slot 0 and that id's processed logit in slot 1, beside the usual lse
// partials.  topk > 0 runs the plain partial kernel with K candidates per chunk; sample_tail_kernel merges them to the
// row's top K and draws the noise of those.  sample_tail_kernel (one warp per row) then does the bookkeeping above and
// the step advance; search_init_kernel<false, true> also resets the per-row hypotheses.
#include "decoder.cuh"

namespace wisb {

namespace {

__device__ __forceinline__ unsigned f2ord(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
// larger key == better candidate: higher score first, then lower index
__device__ __forceinline__ unsigned long long pack_key(float score, unsigned idx) {
  return (static_cast<unsigned long long>(f2ord(score)) << 32) | static_cast<unsigned long long>(~idx);
}

// word 0 of Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11) of counter (c0..c3) and
// key (k0, k1)
__device__ __forceinline__ unsigned philox4x32_10_w0(unsigned c0, unsigned c1, unsigned c2, unsigned c3, unsigned k0,
                                                    unsigned k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const unsigned hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const unsigned hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}

// the Gumbel noise of token v for hypothesis k at generated-token index gen of a window with this seed
__device__ __forceinline__ float gumbel_noise(unsigned long long seed, int k, int gen, int v) {
  const unsigned x = philox4x32_10_w0(static_cast<unsigned>(v), static_cast<unsigned>(gen), static_cast<unsigned>(k), 0u,
                                      static_cast<unsigned>(seed), static_cast<unsigned>(seed >> 32));
  const float u = (static_cast<float>(x >> 9) + 0.5f) * 0x1p-23f;  // exact: 24 significant bits at most
  return -logf(-logf(u));
}

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(0xffffffffu, x, o);
    x = y > x ? y : x;
  }
  return x;
}

// cache slot every later step reads the K/V of position pos from, for a row whose step wrote them into slot `own`: a
// position inside the prompt that a prefill pass forwarded lives only in the slot of the window's first row, prefix
__device__ __forceinline__ int kv_slot(const SearchArgs& a, int pos, int prefix, int own) {
  return a.prompt_fed != nullptr && pos < *a.prompt_fed ? prefix : own;
}

__device__ __forceinline__ float masked_logit(const SearchArgs& a, const float* row, int v, bool first_step) {
  const unsigned char m = a.mask[v];
  if ((m & 1) || (first_step && (m & 2))) return -INFINITY;
  return row[v];
}

// Per-row state of the timestamp rules, from the row's own generated tokens seq[*flip][r][0, gen).
struct TsRule {
  int lo, hi;          // timestamps outside [lo, hi] are off (rules 2 and 4)
  int text_off;        // gen == 0: every id < ts_begin is off (rule 2)
  int below_eot_off;   // last token a timestamp, the one before it not: ids < eot are off (rule 3b)
  int ts_off;          // last two tokens timestamps (or gen == 1 after one): timestamps are off (rule 3a)
};

// warp-cooperative: every lane returns the same state
__device__ __forceinline__ TsRule ts_rule_state(const SearchArgs& a, int r, int gen) {
  const int lane = threadIdx.x & 31;
  const int* hist = a.seq[*a.flip] + static_cast<long long>(r) * a.max_new;
  int last = -1;  // index of the last timestamp of the history
  for (int t = lane; t < gen; t += 32)
    if (hist[t] >= a.ts_begin) last = t;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
  const bool last_ts = gen >= 1 && hist[gen - 1] >= a.ts_begin;
  const bool pen_ts = gen < 2 || hist[gen - 2] >= a.ts_begin;
  TsRule s;
  s.text_off = gen == 0;
  s.below_eot_off = last_ts && !pen_ts;
  s.ts_off = last_ts && pen_ts;
  s.lo = last >= 0 ? hist[last] + (s.below_eot_off ? 0 : 1) : a.ts_begin;
  s.hi = gen == 0 ? a.ts_max_init : a.n_vocab - 1;
  return s;
}

__device__ __forceinline__ float ts_masked_logit(const SearchArgs& a, const TsRule& s, const float* row, int v, bool first_step) {
  if (v < a.ts_begin) {
    if (s.text_off || v == a.no_ts || (s.below_eot_off && v < a.eot)) return -INFINITY;
  } else if (s.ts_off || v < s.lo || v > s.hi) {
    return -INFINITY;
  }
  return masked_logit(a, row, v, first_step);
}

// block-wide selection of the `n_cand` largest keys among each thread's private keys[0..cnt)
template <int PER>
__device__ void block_select(unsigned long long (&keys)[PER], int n_cand, unsigned long long* out,
                             unsigned long long* s_red /*[32]*/) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nwarps = blockDim.x >> 5;
  for (int c = 0; c < n_cand; ++c) {
    unsigned long long best = 0ull;
    int bi = -1;
#pragma unroll
    for (int i = 0; i < PER; ++i)
      if (keys[i] > best) {
        best = keys[i];
        bi = i;
      }
    unsigned long long wbest = best;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, wbest, o);
      wbest = other > wbest ? other : wbest;
    }
    if (lane == 0) s_red[warp] = wbest;
    __syncthreads();
    unsigned long long bbest = s_red[0];
    for (int w = 1; w < nwarps; ++w) bbest = s_red[w] > bbest ? s_red[w] : bbest;
    __syncthreads();
    if (bi >= 0 && best == bbest && best != 0ull) {  // keys are unique (index is part of the key)
#pragma unroll
      for (int i = 0; i < PER; ++i)
        if (i == bi) keys[i] = 0ull;
    }
    if (tid == 0) out[c] = bbest;
  }
}

// grid (NCH, R): partial top-n_cand of one chunk of one row.  NCH = TOPK_CHUNKS: the vocabulary in 32 chunks.
// NCH = TOPK_CHUNKS + 1 (timestamp mode): chunks 0..31 split the text ids [0, ts_begin), chunk 32 holds the timestamps.
constexpr int TK_THREADS = 256;
constexpr int TK_PER = 8;  // 256 * 8 = 2048 >= ceil(51865 / 32) = 1621 and >= the 1501 timestamps
constexpr int HIST_MAX = 448;  // generated tokens a row can hold (T_MAX): gen <= max_new - 1 < HIST_MAX

// History flags of the chunk [v0, v1) of row r (every thread of the block): pen[v - v0] = 1 for ids in hist (when the
// penalty is on), ban[v - v0] = 1 for ids the n-gram rule bans.  Ends with a block barrier.
__device__ void hist_flags(const SearchArgs& a, int r, int v0, int v1, int* s_hist, unsigned char* pen, unsigned char* ban) {
  const int tid = threadIdx.x;
  const int gen = a.st->gen_step;
  const int* hist = a.seq[*a.flip] + static_cast<long long>(r) * a.max_new;
  for (int t = tid; t < gen; t += TK_THREADS) s_hist[t] = hist[t];
  for (int i = tid; i < TK_THREADS * TK_PER / 16; i += TK_THREADS) {
    reinterpret_cast<uint4*>(pen)[i] = make_uint4(0u, 0u, 0u, 0u);
    reinterpret_cast<uint4*>(ban)[i] = make_uint4(0u, 0u, 0u, 0u);
  }
  __syncthreads();
  if (a.rep_penalty != 1.f)
    for (int t = tid; t < gen; t += TK_THREADS) {
      const int v = s_hist[t];
      if (v >= v0 && v < v1) pen[v - v0] = 1;  // duplicates store the same byte: penalised once
    }
  const int n = a.no_repeat_ngram;
  if (n > 0)  // (no n-gram is complete while gen < n: the loop is empty, which covers transformers' gen + 1 < n guard)
    for (int i = tid; i <= gen - n; i += TK_THREADS) {
      bool same = true;
      for (int j = 0; j < n - 1 && same; ++j) same = s_hist[i + j] == s_hist[gen - n + 1 + j];
      const int v = s_hist[i + n - 1];
      if (same && v >= v0 && v < v1) ban[v - v0] = 1;
    }
  __syncthreads();
}

// the history processors on a logit that already went through the masks (a masked id stays -inf)
__device__ __forceinline__ float hist_logit(const SearchArgs& a, float x, unsigned char pen, unsigned char ban) {
  if (pen) x = x < 0.f ? x * a.rep_penalty : x / a.rep_penalty;
  return ban ? -INFINITY : x;
}

template <int NCH, bool HIST, bool SAMPLE = false>
__global__ void __launch_bounds__(TK_THREADS) topk_partial_kernel(const SearchArgs a) {
  // Within one row the ranking by processed logit equals the ranking by score, so the per-chunk stage needs no
  // log-sum-exp: it emits the chunk's top-n_cand logits plus (max, sum exp) partials; the merge stage turns them into
  // the row's lse and into scores, with no separate two-pass lse kernel.  SAMPLE (sampling over the whole vocabulary):
  // the chunk's best Gumbel key instead of its top logits.
  constexpr bool TS = NCH > TOPK_CHUNKS;
  __shared__ unsigned long long s_red[32];
  __shared__ float s_f[32];
  __shared__ TsRule s_rule;
  if (a.st->all_done) return;  // a step enqueued ahead of the host's poll
  const int chunk = blockIdx.x, r = blockIdx.y;
  const bool first = a.st->gen_step == 0;
  // the first step after a prefill pass that also produced the logits reads the window's row of its last prompt position
  const long long lrow = first && a.prompt_fed != nullptr && *a.prompt_fed == a.prompt_len
                             ? static_cast<long long>(r / a.beam) * a.prompt_len + a.prompt_len - 1
                             : r;
  const float* row = a.logits + lrow * a.ldl;
  int v0, v1;
  if (!TS) {
    const int per_chunk = (a.n_vocab + TOPK_CHUNKS - 1) / TOPK_CHUNKS;
    v0 = chunk * per_chunk;
    v1 = min(a.n_vocab, v0 + per_chunk);
  } else if (chunk < TOPK_CHUNKS) {
    const int per_chunk = (a.ts_begin + TOPK_CHUNKS - 1) / TOPK_CHUNKS;
    v0 = chunk * per_chunk;
    v1 = min(a.ts_begin, v0 + per_chunk);
  } else {
    v0 = a.ts_begin;
    v1 = a.n_vocab;
  }
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned char* pen = nullptr;
  const unsigned char* ban = nullptr;
  if constexpr (HIST) {
    __shared__ int s_hist[HIST_MAX];
    __shared__ __align__(16) unsigned char s_pen[TK_THREADS * TK_PER];
    __shared__ __align__(16) unsigned char s_ban[TK_THREADS * TK_PER];
    hist_flags(a, r, v0, v1, s_hist, s_pen, s_ban);
    pen = s_pen;
    ban = s_ban;
  }
  TsRule rule;
  if (TS) {
    if (warp == 0) {
      const TsRule t = ts_rule_state(a, r, a.st->gen_step);
      if (lane == 0) s_rule = t;
    }
    __syncthreads();
    rule = s_rule;
  }
  unsigned long long keys[TK_PER];
  float lg[TK_PER];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < TK_PER; ++i) {
    const int v = v0 + tid + i * TK_THREADS;
    keys[i] = 0ull;
    lg[i] = -INFINITY;
    if (v < v1) {
      lg[i] = TS ? ts_masked_logit(a, rule, row, v, first) : masked_logit(a, row, v, first);
      if constexpr (HIST) lg[i] = hist_logit(a, lg[i], pen[v - v0], ban[v - v0]);
      if (lg[i] != -INFINITY) keys[i] = pack_key(lg[i], static_cast<unsigned>(v));
      mx = fmaxf(mx, lg[i]);
    }
  }
  mx = warp_max(mx);
  if (lane == 0) s_f[warp] = mx;
  __syncthreads();
  mx = s_f[0];
  for (int w = 1; w < TK_THREADS / 32; ++w) mx = fmaxf(mx, s_f[w]);
  __syncthreads();
  float se = 0.f;
#pragma unroll
  for (int i = 0; i < TK_PER; ++i)
    if (lg[i] != -INFINITY) se += __expf(lg[i] - mx);
  se = warp_sum(se);
  if (lane == 0) s_f[warp] = se;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
    for (int w = 0; w < TK_THREADS / 32; ++w) t += s_f[w];
    a.part_max[r * NCH + chunk] = mx;
    a.part_sum[r * NCH + chunk] = t;
  }
  if constexpr (SAMPLE) {
    // the chunk's largest key fp32(l / T) + g (ties: lowest id) -> part slot 0, packed; its processed logit -> slot 1
    __shared__ float s_l[32];
    const int u = r / a.beam, k = r - u * a.beam, gen = a.st->gen_step;
    const unsigned long long seed = a.seed_u[u];
    unsigned long long best = 0ull;
    float best_l = -INFINITY;
#pragma unroll
    for (int i = 0; i < TK_PER; ++i) {
      if (lg[i] == -INFINITY) continue;
      const int v = v0 + tid + i * TK_THREADS;
      const float key = __fdiv_rn(lg[i], a.temperature) + gumbel_noise(seed, k, gen, v);
      const unsigned long long pk = pack_key(key, static_cast<unsigned>(v));
      if (pk > best) {
        best = pk;
        best_l = lg[i];
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ob = __shfl_xor_sync(0xffffffffu, best, o);
      const float ol = __shfl_xor_sync(0xffffffffu, best_l, o);
      if (ob > best) {
        best = ob;
        best_l = ol;
      }
    }
    if (lane == 0) {
      s_red[warp] = best;
      s_l[warp] = best_l;
    }
    __syncthreads();
    if (tid == 0) {  // (holds warp 0's best already)
      for (int w = 1; w < TK_THREADS / 32; ++w)
        if (s_red[w] > best) {
          best = s_red[w];
          best_l = s_l[w];
        }
      unsigned long long* out = a.part + (static_cast<long long>(r) * NCH + chunk) * MAX_CAND;
      out[0] = best;
      out[1] = __float_as_uint(best_l);
    }
    return;
  }
  block_select<TK_PER>(keys, a.n_cand, a.part + (static_cast<long long>(r) * NCH + chunk) * MAX_CAND, s_red);
}

// grid (n_utt): merge beam * NCH * n_cand partial keys -> sorted candidate list
template <int NCH>
constexpr int tm_per() { return (MAX_BEAM * NCH * MAX_CAND + TK_THREADS - 1) / TK_THREADS; }  // 16 / 17

template <int NCH, bool MIXED>
__device__ __forceinline__ void topk_merge_body(const SearchArgs& a, unsigned long long* s_red, unsigned long long* s_out,
                                                float* s_lse, int* s_ts_only) {
  constexpr bool TS = NCH > TOPK_CHUNKS;
  constexpr int TM_PER = tm_per<NCH>();
  const int u = blockIdx.x;
  const int gen = a.st->gen_step;
  const bool first = gen == 0;
  // rows of the utterance's block that it searches, candidates it keeps, its length penalty (MIXED: its own)
  const int beam = MIXED ? a.beam_u[u] : a.beam;
  const int n_cand = MIXED ? 2 * beam : a.n_cand;
  const float lp = MIXED ? a.lp_u[u] : a.length_penalty;
  const float norm = (lp != 0.f) ? powf(static_cast<float>(gen + 1), lp) : 1.f;
  if (threadIdx.x < beam) {  // row log-sum-exp from the chunk partials
    const int r = u * a.beam + threadIdx.x;
    float mx = -INFINITY;
    for (int c = 0; c < NCH; ++c) mx = fmaxf(mx, a.part_max[r * NCH + c]);
    float t = 0.f;
    for (int c = 0; c < NCH; ++c) {
      const float pm = a.part_max[r * NCH + c];
      if (pm != -INFINITY) t += a.part_sum[r * NCH + c] * __expf(pm - mx);
    }
    float lse = mx + logf(t);
    if (TS) {
      // rule 5: the row's timestamp log-sum-exp against its best text logit (the log-softmax normaliser cancels)
      float text_max = -INFINITY;
      for (int c = 0; c < TOPK_CHUNKS; ++c) text_max = fmaxf(text_max, a.part_max[r * NCH + c]);
      const float pm = a.part_max[r * NCH + TOPK_CHUNKS];
      const float ts_lse = pm == -INFINITY ? -INFINITY : pm + logf(a.part_sum[r * NCH + TOPK_CHUNKS]);
      const int ts_only = ts_lse > text_max;
      s_ts_only[threadIdx.x] = ts_only;
      if (ts_only) lse = ts_lse;
    }
    s_lse[threadIdx.x] = lse;
    a.row_lse[r] = lse;
  }
  __syncthreads();
  const int total = beam * NCH * n_cand;
  unsigned long long keys[TM_PER];
#pragma unroll
  for (int i = 0; i < TM_PER; ++i) {
    const int j = threadIdx.x + i * TK_THREADS;
    keys[i] = 0ull;
    if (j < total) {
      const int c = j % n_cand;          // (MIXED: the chunk's first n_cand of its a.n_cand sorted partials)
      const int rc = j / n_cand;         // (beam row, chunk)
      const int k = rc / NCH;            // beam index
      const unsigned long long pk = a.part[(static_cast<long long>(u * a.beam) * NCH + rc) * MAX_CAND + c];
      // at the first step every beam holds the same prefix: only beam 0 counts
      const bool dropped = TS && s_ts_only[k] && rc % NCH < TOPK_CHUNKS;  // rule 5 turned this row's text off
      if (pk != 0ull && !(first && k > 0) && !dropped) {
        const float lg = ord2f(static_cast<unsigned>(pk >> 32));
        const unsigned v = ~static_cast<unsigned>(pk & 0xffffffffull);
        const float sc = ((lg - s_lse[k]) + a.cum[u * a.beam + k]) / norm;
        keys[i] = pack_key(sc, static_cast<unsigned>(k * a.n_vocab) + v);
      }
    }
  }
  block_select<TM_PER>(keys, n_cand, s_out, s_red);
  __syncthreads();
  if (threadIdx.x < a.n_cand) {  // (MIXED: entries n_cand .. a.n_cand - 1 are none)
    const unsigned long long key = s_out[threadIdx.x];
    const bool valid = key != 0ull && (!MIXED || static_cast<int>(threadIdx.x) < n_cand);
    a.cand_score[u * MAX_CAND + threadIdx.x] = valid ? ord2f(static_cast<unsigned>(key >> 32)) : -INFINITY;
    a.cand_idx[u * MAX_CAND + threadIdx.x] = valid ? static_cast<int>(~static_cast<unsigned>(key & 0xffffffffull)) : -1;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// one warp: the CTranslate2 bookkeeping for one utterance
template <bool MIXED>
__device__ __forceinline__ void search_bookkeeping_body(const SearchArgs& a, int* s_pick, int& s_best_k, int& s_finished) {
  const int u = blockIdx.x, lane = threadIdx.x;
  const int rows = a.beam;  // row block of an utterance
  const int beam = MIXED ? a.beam_u[u] : a.beam, V = a.n_vocab, nc = MIXED ? 2 * beam : a.n_cand;
  const int gen = a.st->gen_step, pos = a.st->pos;
  const int cur = *a.flip, nxt_buf = cur ^ 1;
  const int* seq_cur = a.seq[cur];
  int* seq_nxt = a.seq[nxt_buf];
  const int* ind_cur = a.indir[cur];
  int* ind_nxt = a.indir[nxt_buf];

  if (a.done[u]) {
    // frozen utterance: carry the state over unchanged so the ping-pong buffers stay coherent
    for (int k = 0; k < rows; ++k) {
      const int r = u * rows + k;
      for (int t = lane; t < a.max_new; t += 32) seq_nxt[r * a.max_new + t] = seq_cur[r * a.max_new + t];
      for (int t = lane; t < a.t_max; t += 32)
        ind_nxt[r * a.t_max + t] = (t == pos) ? kv_slot(a, pos, u * rows, r) : ind_cur[r * a.t_max + t];
    }
    return;
  }
  const float* cs = a.cand_score + u * MAX_CAND;
  const int* ci = a.cand_idx + u * MAX_CAND;
  const int cap = a.max_new_u != nullptr ? a.max_new_u[u] : a.max_new;
  const bool is_last = gen + 1 >= cap;
  const bool capped = gen >= cap;  // a cap of 0 new tokens: the utterance finishes without a hypothesis
  const float lp = MIXED ? a.lp_u[u] : a.length_penalty;
  const float norm = (lp != 0.f) ? powf(static_cast<float>(gen + 1), lp) : 1.f;
  if (lane == 0) {
    int n_hyp = a.n_hyp[u];
    float best = a.best_score[u];
    int best_k = -1;
    int secondary = beam;
    for (int k = 0; k < beam; ++k) {
      int pick = k;
      const int idx = ci[k];
      const int tok = idx < 0 ? a.eot : idx % V;
      if (!capped && idx >= 0 && (tok == a.eot || is_last)) {
        ++n_hyp;
        if (cs[k] > best) {  // strict: the first best hypothesis wins ties
          best = cs[k];
          best_k = k;
        }
        for (int j = secondary; j < nc; ++j) {
          if (ci[j] >= 0 && ci[j] % V != a.eot) {
            pick = j;
            secondary = j + 1;
            break;
          }
        }
      }
      s_pick[k] = pick;
    }
    a.n_hyp[u] = n_hyp;
    a.best_score[u] = best;
    s_best_k = best_k;
    const int fin = (is_last || n_hyp >= (MIXED ? a.max_hyp_u[u] : a.max_hyp)) ? 1 : 0;
    s_finished = fin;
    if (fin) {
      a.done[u] = 1;
      atomicAdd(&a.st->n_done, 1);  // all_done follows in the step advance, once every CTA has taken its ticket
    }
  }
  __syncwarp();
  if (s_best_k >= 0) {  // record the new best hypothesis (tokens of its parent beam + the last token unless eot)
    const int k = s_best_k;
    const int idx = ci[k];
    const int parent = idx / V, tok = idx % V;
    const int pr = u * rows + parent;
    for (int t = lane; t < gen; t += 32) a.best_tokens[u * a.max_new + t] = seq_cur[pr * a.max_new + t];
    if (lane == 0) {
      int len = gen;
      if (tok != a.eot) {
        a.best_tokens[u * a.max_new + gen] = tok;
        len = gen + 1;
      }
      a.best_len[u] = len;
    }
  }
  // next alive beams (also written when finished: harmless, keeps buffers defined); a row the utterance does not search
  // carries itself over as a dead row
  for (int k = 0; k < rows; ++k) {
    const int r = u * rows + k;
    const int idx = (!MIXED || k < beam) ? ci[s_pick[k]] : -1;
    const int parent = idx < 0 ? k : idx / V;
    const int tok = idx < 0 ? a.eot : idx % V;
    const int pr = u * rows + parent;
    for (int t = lane; t < gen; t += 32) seq_nxt[r * a.max_new + t] = seq_cur[pr * a.max_new + t];
    for (int t = lane; t < pos; t += 32) ind_nxt[r * a.t_max + t] = ind_cur[pr * a.t_max + t];
    if (lane == 0) {
      if (gen < a.max_new) seq_nxt[r * a.max_new + gen] = tok;
      ind_nxt[r * a.t_max + pos] = kv_slot(a, pos, u * rows, pr);  // this step's K/V: the parent row's own slot
      a.tokens[r] = tok;
      a.cum[r] = (idx < 0) ? -INFINITY : cs[s_pick[k]] * norm;
    }
  }
}

// End of a search tail launch (every thread, after a barrier that follows the CTA's bookkeeping): the last CTA to take a
// ticket advances the step (position, generation step, ping-pong flip, per-row positions) and sets all_done.
__device__ __forceinline__ void step_advance(const SearchArgs& a, int& s_last) {
  if (threadIdx.x == 0) {
    __threadfence();
    const int t = atomicAdd(&a.st->ticket, 1);
    s_last = t == static_cast<int>(gridDim.x) - 1;
  }
  __syncthreads();
  if (s_last) {  // every utterance has read this step's position / generation step / flip
    if (threadIdx.x == 0) {
      // set here, not by the CTA that finishes the last utterance: a CTA of this launch that starts after that one
      // must still take its ticket, or the advance below is skipped
      if (atomicAdd(&a.st->n_done, 0) == a.n_utt) a.st->all_done = 1;
      a.st->ticket = 0;
      a.st->pos += 1;
      a.st->gen_step += 1;
      *a.flip ^= 1;
    }
    if (a.row_pos != nullptr)
      for (int i = threadIdx.x; i < a.n_utt * a.beam; i += blockDim.x) a.row_pos[i] += 1;
  }
}

// grid (n_utt) x TK_THREADS: candidate merge, then (warp 0) the bookkeeping of the utterance, then -- by the last CTA to get
// there -- the step advance (position, generation step, ping-pong flip, per-row positions).  One launch instead of three:
// the tail of a decoding step is launch-latency bound.
template <int NCH, bool MIXED>
__global__ void __launch_bounds__(TK_THREADS) search_tail_kernel(const SearchArgs a) {
  __shared__ unsigned long long s_red[32];
  __shared__ unsigned long long s_out[MAX_CAND];
  __shared__ float s_lse[MAX_BEAM];
  __shared__ int s_ts_only[MAX_BEAM];
  __shared__ int s_pick[MAX_BEAM];
  __shared__ int s_best_k;
  __shared__ int s_finished;
  __shared__ int s_last;
  if (a.st->all_done) return;  // a step enqueued ahead of the host's poll: nothing left to do
  topk_merge_body<NCH, MIXED>(a, s_red, s_out, s_lse, s_ts_only);
  __syncthreads();  // the candidate list (global) is complete for this CTA's readers
  if (threadIdx.x < 32) search_bookkeeping_body<MIXED>(a, s_pick, s_best_k, s_finished);
  __syncthreads();
  step_advance(a, s_last);
}

// grid (n_utt) x TK_THREADS, sampling: warp k does hypothesis row k of the utterance (selection from the chunk partials,
// then its bookkeeping), thread 0 decides whether the utterance is done, then the step advance of search_tail_kernel.
template <int NCH>
__global__ void __launch_bounds__(TK_THREADS) sample_tail_kernel(const SearchArgs a) {
  constexpr bool TS = NCH > TOPK_CHUNKS;
  constexpr int PER = (NCH * MAX_CAND + 31) / 32;  // a row's chunk partials per lane (topk > 0): 16 / 17
  __shared__ int s_live[MAX_BEAM];
  __shared__ int s_last;
  if (a.st->all_done) return;  // a step enqueued ahead of the host's poll: nothing left to do
  const int u = blockIdx.x, k = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = a.beam, r = u * n + k;
  const int gen = a.st->gen_step, pos = a.st->pos;
  const int cur = *a.flip;
  const bool frozen = a.done[u] != 0;  // (written below only after a barrier)
  const int cap = a.max_new_u != nullptr ? a.max_new_u[u] : a.max_new;
  const bool is_last = gen + 1 >= cap;
  const bool capped = gen >= cap;  // a cap of 0 new tokens: the utterance finishes without a hypothesis
  if (k < n) {
    const int* seq_cur = a.seq[cur] + static_cast<long long>(r) * a.max_new;
    int* seq_nxt = a.seq[cur ^ 1] + static_cast<long long>(r) * a.max_new;
    const int* ind_cur = a.indir[cur] + static_cast<long long>(r) * a.t_max;
    int* ind_nxt = a.indir[cur ^ 1] + static_cast<long long>(r) * a.t_max;
    // rows never reorder: the history and the cache indirection carry over, this step's K/V are the row's own (kv_slot)
    for (int t = lane; t < gen; t += 32) seq_nxt[t] = seq_cur[t];
    for (int t = lane; t < pos; t += 32) ind_nxt[t] = ind_cur[t];
    // row log-sum-exp from the chunk partials (every lane), rule 5 as in topk_merge_body
    float mx = -INFINITY;
    for (int c = 0; c < NCH; ++c) mx = fmaxf(mx, a.part_max[r * NCH + c]);
    float t = 0.f;
    for (int c = 0; c < NCH; ++c) {
      const float pm = a.part_max[r * NCH + c];
      if (pm != -INFINITY) t += a.part_sum[r * NCH + c] * __expf(pm - mx);
    }
    float lse = mx + logf(t);
    bool ts_only = false;
    if (TS) {
      float text_max = -INFINITY;
      for (int c = 0; c < TOPK_CHUNKS; ++c) text_max = fmaxf(text_max, a.part_max[r * NCH + c]);
      const float pm = a.part_max[r * NCH + TOPK_CHUNKS];
      const float ts_lse = pm == -INFINITY ? -INFINITY : pm + logf(a.part_sum[r * NCH + TOPK_CHUNKS]);
      ts_only = ts_lse > text_max;
      if (ts_only) lse = ts_lse;
    }
    const float cum = a.cum[r];
    const bool live = !frozen && !capped && cum != -INFINITY;
    unsigned long long best = 0ull;  // packed (key, ~id) of the sampled token, 0 = none
    float best_l = -INFINITY;        // its processed logit
    if (live) {
      const unsigned long long* part = a.part + static_cast<long long>(r) * NCH * MAX_CAND;
      if (a.topk == 0) {
        unsigned long long pk = 0ull;  // the lane's best chunk key (chunks lane and lane + 32)
        int pc = 0;
        for (int c = lane; c < NCH; c += 32) {
          const unsigned long long q = (TS && ts_only && c < TOPK_CHUNKS) ? 0ull : part[c * MAX_CAND];
          if (q > pk) {
            pk = q;
            pc = c;
          }
        }
        best = warp_max_u64(pk);
        const unsigned owner = __ballot_sync(0xffffffffu, pk == best && best != 0ull);
        const int c_best = __shfl_sync(0xffffffffu, pc, owner ? __ffs(owner) - 1 : 0);
        if (best != 0ull) best_l = __uint_as_float(static_cast<unsigned>(part[c_best * MAX_CAND + 1]));
      } else {
        // the row's top-K processed logits from the chunks' sorted top K (lane i keeps the i-th), then their keys
        const int K = a.topk;
        unsigned long long e[PER];
#pragma unroll
        for (int i = 0; i < PER; ++i) {
          const int j = lane + 32 * i, c = j / K;
          e[i] = 0ull;
          if (j < NCH * K && !(TS && ts_only && c < TOPK_CHUNKS)) e[i] = part[c * MAX_CAND + (j - c * K)];
        }
        unsigned long long mine = 0ull;
        for (int s = 0; s < K; ++s) {
          unsigned long long m = 0ull;
#pragma unroll
          for (int i = 0; i < PER; ++i) m = e[i] > m ? e[i] : m;
          m = warp_max_u64(m);
          if (m == 0ull) break;  // (warp-uniform) fewer than K finite logits
#pragma unroll
          for (int i = 0; i < PER; ++i)
            if (e[i] == m) e[i] = 0ull;  // keys are unique (the id is part of the key)
          if (lane == s) mine = m;
        }
        unsigned long long pk = 0ull;
        float lm = -INFINITY;
        if (mine != 0ull) {
          lm = ord2f(static_cast<unsigned>(mine >> 32));
          const unsigned v = ~static_cast<unsigned>(mine & 0xffffffffull);
          const float key = __fdiv_rn(lm, a.temperature) + gumbel_noise(a.seed_u[u], k, gen, static_cast<int>(v));
          pk = pack_key(key, v);
        }
        best = warp_max_u64(pk);
        const unsigned owner = __ballot_sync(0xffffffffu, pk == best && best != 0ull);
        best_l = __shfl_sync(0xffffffffu, lm, owner ? __ffs(owner) - 1 : 0);
      }
    }
    const bool has = best != 0ull;
    const int tok = has ? static_cast<int>(~static_cast<unsigned>(best & 0xffffffffull)) : a.eot;
    const float cum_new = has ? (best_l - lse) + cum : -INFINITY;
    const bool finish = has && (tok == a.eot || is_last);
    if (finish)  // the hypothesis: the row's tokens, plus the last one unless eot
      for (int t2 = lane; t2 < gen; t2 += 32) a.best_tokens[static_cast<long long>(r) * a.max_new + t2] = seq_cur[t2];
    if (lane == 0) {
      a.row_lse[r] = lse;
      if (gen < a.max_new) seq_nxt[gen] = tok;
      ind_nxt[pos] = kv_slot(a, pos, u * n, r);
      if (finish) {
        int len = gen;
        if (tok != a.eot) {
          a.best_tokens[static_cast<long long>(r) * a.max_new + gen] = tok;
          len = gen + 1;
        }
        const float lp = a.length_penalty;
        const float norm = (lp != 0.f) ? powf(static_cast<float>(gen + 1), lp) : 1.f;
        a.best_len[r] = len;
        a.best_score[r] = cum_new / norm;
      }
      const bool cont = has && !finish;
      a.tokens[r] = cont ? tok : a.eot;
      a.cum[r] = cont ? cum_new : -INFINITY;
      a.cand_idx[u * MAX_CAND + k] = has ? tok : -1;
      a.cand_score[u * MAX_CAND + k] = has ? ord2f(static_cast<unsigned>(best >> 32)) : -INFINITY;
      s_live[k] = cont ? 1 : 0;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && !frozen) {
    int any = 0;
    for (int j = 0; j < n; ++j) any |= s_live[j];
    if (!any) {  // (at the last step, or capped, no row continues)
      a.done[u] = 1;
      atomicAdd(&a.st->n_done, 1);
    }
  }
  __syncthreads();
  step_advance(a, s_last);
}

__global__ void prefill_rows_kernel(int* tokens, int* row_pos, int* row_slot, const int* prompt, int prompt_len, int rows,
                                    int p0, int chunk, int beam) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  const int u = i / chunk, p = p0 + i % chunk;
  tokens[i] = prompt[u * prompt_len + p];
  row_pos[i] = p;
  row_slot[i] = u * beam;
}

__global__ void prefill_advance_kernel(int* tokens, const int* prompt, int prompt_len, int R, int beam, DecState* st) {
  const int next = st->pos + 1;
  for (int r = threadIdx.x; r < R; r += blockDim.x) tokens[r] = prompt[(r / beam) * prompt_len + next];
  __syncthreads();
  if (threadIdx.x == 0) st->pos = next;
}

// fed > 0: prompt positions [0, fed) were forwarded once per utterance into the cache slot of its first beam by a single
// prefill pass; decoding then starts at the last prompt token (fed = prompt_len: that pass also produced its logits, so
// the first step runs no pass) and every beam's indirection points at that slot.  MIXED: rows an utterance does not
// search start dead (eot, cum -inf).  SAMPLE: every row is live and has no hypothesis yet (the per-row best_len /
// best_score).
template <bool MIXED, bool SAMPLE = false>
__global__ void search_init_kernel(const SearchArgs a, const int* prompt, int fed) {
  const int R = a.n_utt * a.beam;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, n = gridDim.x * blockDim.x;
  const int pos0 = min(fed, a.prompt_len - 1);
  if (tid == 0) {
    a.st->pos = pos0;
    a.st->gen_step = 0;
    a.st->n_done = 0;
    a.st->all_done = 0;
    a.st->ticket = 0;
    *a.flip = 0;
    if (a.prompt_fed != nullptr) *a.prompt_fed = fed;
  }
  for (int i = tid; i < R; i += n) {
    const bool dead = MIXED && i % a.beam >= a.beam_u[i / a.beam];
    a.tokens[i] = dead ? a.eot : prompt[(i / a.beam) * a.prompt_len + pos0];
    a.cum[i] = dead ? -INFINITY : 0.f;
    if (a.row_pos != nullptr) {
      a.row_pos[i] = pos0;
      a.row_slot[i] = i;
    }
  }
  for (int i = tid; i < a.n_utt; i += n) {
    a.done[i] = 0;
    a.n_hyp[i] = 0;
    a.best_score[i] = -INFINITY;
    a.best_len[i] = 0;
  }
  if constexpr (SAMPLE)
    for (int i = tid; i < R; i += n) {
      a.best_score[i] = -INFINITY;
      a.best_len[i] = 0;
    }
  for (int i = tid; i < R * a.t_max; i += n) {
    const int r = i / a.t_max;
    const int slot = fed > 0 ? (r / a.beam) * a.beam : r;  // else identity: every row holds its own prefix copy
    a.indir[0][i] = slot;
    a.indir[1][i] = slot;
  }
}

__global__ void lang_probs_kernel(const float* logits, long long ldl, const int* lang_ids, int n_lang, int row_stride,
                                  float* probs) {
  __shared__ float s_v[128];
  const int u = blockIdx.x;
  const float* row = logits + static_cast<long long>(u) * row_stride * ldl;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < n_lang; i += blockDim.x) {
    s_v[i] = row[lang_ids[i]];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 0; i < n_lang; ++i) mx = fmaxf(mx, s_v[i]);
    float s = 0.f;
    for (int i = 0; i < n_lang; ++i) s += expf(s_v[i] - mx);
    for (int i = 0; i < n_lang; ++i) probs[u * n_lang + i] = expf(s_v[i] - mx) / s;
  }
}

constexpr int NS_THREADS = 256;

// sum (ADD) or max over the CTA; every thread gets the result
template <bool ADD>
__device__ float ns_block_reduce(float v, float* s_red) {
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = ADD ? v + w : fmaxf(v, w);
  }
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = s_red[0];
  for (int i = 1; i < NS_THREADS / 32; ++i) v = ADD ? v + s_red[i] : fmaxf(v, s_red[i]);
  __syncthreads();  // (s_red is reused by the next reduction)
  return v;
}

// CTA u: out[u] = softmax(row)[no_speech] over columns [0, n_vocab) of logits row rows[u]; rows[u] < 0 leaves out[u]
__global__ void __launch_bounds__(NS_THREADS) no_speech_kernel(const float* logits, long long ldl, const int* rows,
                                                               int n_vocab, int no_speech, float* out) {
  __shared__ float s_red[NS_THREADS / 32];
  const int u = blockIdx.x, r = rows[u];
  if (r < 0) return;
  const float* row = logits + static_cast<long long>(r) * ldl;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < n_vocab; i += NS_THREADS) mx = fmaxf(mx, row[i]);
  mx = ns_block_reduce<false>(mx, s_red);
  float s = 0.f;
  for (int i = threadIdx.x; i < n_vocab; i += NS_THREADS) s += expf(row[i] - mx);
  s = ns_block_reduce<true>(s, s_red);
  if (threadIdx.x == 0) out[u] = expf(row[no_speech] - mx) / s;
}

// CTA u: dst row u = src row rows[u] (d fp16 values, d % 8 == 0); rows[u] < 0 leaves dst row u
__global__ void __launch_bounds__(128) row_gather_kernel(const __half* src, int d, const int* rows, __half* dst) {
  const int u = blockIdx.x, r = rows[u];
  if (r < 0) return;
  const uint4* s = reinterpret_cast<const uint4*>(src + static_cast<long long>(r) * d);
  uint4* t = reinterpret_cast<uint4*>(dst + static_cast<long long>(u) * d);
  for (int i = threadIdx.x; i < d / 8; i += blockDim.x) t[i] = s[i];
}

}  // namespace

void search_step_run(const SearchArgs& a, cudaStream_t stream) {
  const int R = a.n_utt * a.beam;
  WISB_REQUIRE(a.beam >= 1 && a.beam <= MAX_BEAM && a.n_cand <= MAX_CAND, "search: beam_size must be in [1, 8]");
  WISB_REQUIRE((a.n_vocab + TOPK_CHUNKS - 1) / TOPK_CHUNKS <= TK_THREADS * TK_PER, "search: vocabulary too large");
  if (a.ts)
    WISB_REQUIRE(a.ts_begin > a.eot && a.ts_begin < a.n_vocab && a.n_vocab - a.ts_begin <= TK_THREADS * TK_PER &&
                     a.ts_max_init >= a.ts_begin && a.max_new >= 1,
                 "search: bad timestamp geometry");
  const bool hist = a.rep_penalty != 1.f || a.no_repeat_ngram > 0;
  WISB_REQUIRE(!hist || (a.max_new <= HIST_MAX && a.rep_penalty > 0.f && a.no_repeat_ngram >= 0),
               "search: bad history processor arguments");
  const bool mixed = a.beam_u != nullptr;
  WISB_REQUIRE(!mixed || (a.max_hyp_u != nullptr && a.lp_u != nullptr), "search: per-utterance options come as a set");
  if (a.sample) {
    WISB_REQUIRE(!mixed && a.seed_u != nullptr && (a.topk == 0 || (a.topk >= 2 && a.topk <= MAX_CAND)) &&
                     std::isfinite(a.temperature) && a.temperature > 0.f,
                 "search: bad sampling arguments");
    SearchArgs b = a;
    b.n_cand = a.topk;  // topk > 0: the plain partial kernel emits each chunk's top K logits
    const dim3 grid(a.ts ? TOPK_CHUNKS + 1 : TOPK_CHUNKS, R);
    if (a.ts) {
      if (a.topk == 0)
        hist ? topk_partial_kernel<TOPK_CHUNKS + 1, true, true><<<grid, TK_THREADS, 0, stream>>>(b)
             : topk_partial_kernel<TOPK_CHUNKS + 1, false, true><<<grid, TK_THREADS, 0, stream>>>(b);
      else
        hist ? topk_partial_kernel<TOPK_CHUNKS + 1, true><<<grid, TK_THREADS, 0, stream>>>(b)
             : topk_partial_kernel<TOPK_CHUNKS + 1, false><<<grid, TK_THREADS, 0, stream>>>(b);
      sample_tail_kernel<TOPK_CHUNKS + 1><<<a.n_utt, TK_THREADS, 0, stream>>>(b);
    } else {
      if (a.topk == 0)
        hist ? topk_partial_kernel<TOPK_CHUNKS, true, true><<<grid, TK_THREADS, 0, stream>>>(b)
             : topk_partial_kernel<TOPK_CHUNKS, false, true><<<grid, TK_THREADS, 0, stream>>>(b);
      else
        hist ? topk_partial_kernel<TOPK_CHUNKS, true><<<grid, TK_THREADS, 0, stream>>>(b)
             : topk_partial_kernel<TOPK_CHUNKS, false><<<grid, TK_THREADS, 0, stream>>>(b);
      sample_tail_kernel<TOPK_CHUNKS><<<a.n_utt, TK_THREADS, 0, stream>>>(b);
    }
    WISB_CUDA(cudaGetLastError());
    return;
  }
  if (a.ts) {
    if (hist)
      topk_partial_kernel<TOPK_CHUNKS + 1, true><<<dim3(TOPK_CHUNKS + 1, R), TK_THREADS, 0, stream>>>(a);
    else
      topk_partial_kernel<TOPK_CHUNKS + 1, false><<<dim3(TOPK_CHUNKS + 1, R), TK_THREADS, 0, stream>>>(a);
    if (mixed)
      search_tail_kernel<TOPK_CHUNKS + 1, true><<<a.n_utt, TK_THREADS, 0, stream>>>(a);
    else
      search_tail_kernel<TOPK_CHUNKS + 1, false><<<a.n_utt, TK_THREADS, 0, stream>>>(a);
  } else {
    if (hist)
      topk_partial_kernel<TOPK_CHUNKS, true><<<dim3(TOPK_CHUNKS, R), TK_THREADS, 0, stream>>>(a);
    else
      topk_partial_kernel<TOPK_CHUNKS, false><<<dim3(TOPK_CHUNKS, R), TK_THREADS, 0, stream>>>(a);
    if (mixed)
      search_tail_kernel<TOPK_CHUNKS, true><<<a.n_utt, TK_THREADS, 0, stream>>>(a);
    else
      search_tail_kernel<TOPK_CHUNKS, false><<<a.n_utt, TK_THREADS, 0, stream>>>(a);
  }
  WISB_CUDA(cudaGetLastError());
}

void prefill_rows_run(int* tokens, int* row_pos, int* row_slot, const int* prompt, int prompt_len, int n_utt, int p0,
                      int chunk, int beam, cudaStream_t stream) {
  const int rows = n_utt * chunk;
  prefill_rows_kernel<<<cdiv(rows, 256), 256, 0, stream>>>(tokens, row_pos, row_slot, prompt, prompt_len, rows, p0, chunk, beam);
  WISB_CUDA(cudaGetLastError());
}

void prefill_advance_run(int* tokens, const int* prompt, int prompt_len, int R, int beam, DecState* st, cudaStream_t stream) {
  prefill_advance_kernel<<<1, 64, 0, stream>>>(tokens, prompt, prompt_len, R, beam, st);
  WISB_CUDA(cudaGetLastError());
}

void search_init_run(const SearchArgs& a, const int* prompt, cudaStream_t stream, int fed) {
  WISB_REQUIRE(fed >= 0 && fed <= a.prompt_len, "search: more prompt positions forwarded than the prompt has");
  if (a.sample)
    search_init_kernel<false, true><<<8, 256, 0, stream>>>(a, prompt, fed);
  else if (a.beam_u != nullptr)
    search_init_kernel<true><<<8, 256, 0, stream>>>(a, prompt, fed);
  else
    search_init_kernel<false><<<8, 256, 0, stream>>>(a, prompt, fed);
  WISB_CUDA(cudaGetLastError());
}

void lang_probs_run(const float* logits, long long ldl, const int* lang_ids, int n_lang, int n_utt, int row_stride,
                    float* probs, cudaStream_t stream) {
  WISB_REQUIRE(n_lang <= 128, "detect_language: more than 128 language ids");
  lang_probs_kernel<<<n_utt, 128, 0, stream>>>(logits, ldl, lang_ids, n_lang, row_stride, probs);
  WISB_CUDA(cudaGetLastError());
}

void no_speech_run(const float* logits, long long ldl, const int* rows, int n_utt, int n_vocab, int no_speech, float* out,
                   cudaStream_t stream) {
  WISB_REQUIRE(n_vocab >= 1 && n_vocab <= ldl && no_speech >= 0 && no_speech < n_vocab, "no-speech: bad vocabulary geometry");
  no_speech_kernel<<<n_utt, NS_THREADS, 0, stream>>>(logits, ldl, rows, n_vocab, no_speech, out);
  WISB_CUDA(cudaGetLastError());
}

void row_gather_run(const __half* src, int d, const int* rows, int n_utt, __half* dst, cudaStream_t stream) {
  WISB_REQUIRE(d % 8 == 0, "row gather: d must be a multiple of 8");
  row_gather_kernel<<<n_utt, 128, 0, stream>>>(src, d, rows, dst);
  WISB_CUDA(cudaGetLastError());
}

}  // namespace wisb
