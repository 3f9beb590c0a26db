// Decoder-side kernel interface (decoder_mega.cu / decoder_batch.cu / search.cu / align.cu).  Token loop of ctranslate2.models.Whisper.generate
// (main.py:687-692; SURVEY.md section 8a rows A10-A14).
#pragma once
#include "common.cuh"
#include "kernels.h"

namespace wisb {

constexpr int DEC_MAX_ROWS = 8;    // rows (utterances x beams) one decoder pass handles
constexpr int MAX_BEAM = 8;
constexpr int MAX_CAND = 2 * MAX_BEAM;
constexpr int TOPK_CHUNKS = 32;

// Everything the captured decode graphs read at run time lives in device memory so one graph serves every step.
struct DecState {
  int pos;        // position of the token being fed this step
  int gen_step;   // 0-based index of the token being generated (valid once pos >= prompt_len - 1)
  int n_done;     // utterances finished
  int all_done;   // n_done == n_utt
  int ticket;     // CTAs of the search tail that finished this step's bookkeeping (the last one advances the step)
};

enum GemvEpi : int {
  GV_STORE = 0,   // out[r, n] = v
  GV_RESID = 1,   // out[r, n] += v
  GV_GELU = 2,    // out[r, n] = gelu(v)
  GV_QKV = 3,     // n < d: q[r, n] = v ; d <= n < 2d: kcache[slot r][pos][n - d] ; else vcache
};

struct SearchArgs {
  // inputs
  const float* logits = nullptr;  // [R, ldl]
  long long ldl = 0;
  int n_vocab = 0;
  const unsigned char* mask = nullptr;  // [V] bit0: suppressed always, bit1: suppressed at the first generated step
  int n_utt = 0, beam = 0, n_cand = 0;
  int max_new = 0, max_hyp = 0, eot = 0, t_max = 0, prompt_len = 0;
  float length_penalty = 1.f;
  // timestamp mode (the prompt has no <|notimestamps|>): ids in [ts_begin, n_vocab) are timestamps,
  // ts_begin = no_ts + 1; ts_max_init = ts_begin + max_initial_timestamp_index, the last one allowed at the first step
  int ts = 0, ts_begin = 0, no_ts = 0, ts_max_init = 0;
  // workspaces / state (device); NCH = TOPK_CHUNKS chunks per row, TOPK_CHUNKS + 1 in timestamp mode
  float* row_lse = nullptr;       // [R]
  float* part_max = nullptr;      // [R][NCH] chunk max of the processed logits
  float* part_sum = nullptr;      // [R][NCH] chunk sum exp(logit - chunk max)
  float* cum = nullptr;           // [R] cumulative log-prob of the alive beams
  unsigned long long* part = nullptr;  // [R][NCH][MAX_CAND] packed (score, ~index)
  float* cand_score = nullptr;    // [n_utt][MAX_CAND]
  int* cand_idx = nullptr;        // [n_utt][MAX_CAND]   beam * V + token
  int* tokens = nullptr;          // [R] token fed next step
  int* seq[2] = {nullptr, nullptr};    // [R][max_new] generated tokens of the alive beams (ping-pong)
  int* indir[2] = {nullptr, nullptr};  // [R][t_max] cache indirection (ping-pong)
  int* flip = nullptr;            // which of the ping-pong buffers is current (device int)
  int* done = nullptr;            // [n_utt]
  int* n_hyp = nullptr;           // [n_utt]
  float* best_score = nullptr;    // [n_utt]
  int* best_len = nullptr;        // [n_utt]
  int* best_tokens = nullptr;     // [n_utt][max_new]
  DecState* st = nullptr;
  int* row_pos = nullptr;         // [R] position fed by every row this step (batched pass); advanced with st->pos
  int* row_slot = nullptr;        // [R] cache slot every row writes this step's K/V to (= its own row)
  const int* max_new_u = nullptr; // optional [n_utt]: per-utterance cap on generated tokens (<= max_new)
  // history processors on every row's generated tokens (search.cu): 1 / 0 = off
  float rep_penalty = 1.f;        // repetition_penalty, finite and > 0
  int no_repeat_ngram = 0;        // no_repeat_ngram_size, >= 0
  // per-utterance search options (all three or none): utterance u searches rows [0, beam_u[u]) of its block of `beam`
  // rows with 2 * beam_u[u] candidates, max_hyp_u[u] hypotheses and length penalty lp_u[u]; its rows >= beam_u[u] are
  // dead (eot, cum -inf).  `beam` is then the largest of them, `n_cand` 2 * beam; max_hyp / length_penalty are unused.
  const int* beam_u = nullptr;    // [n_utt] in [1, beam]
  const int* max_hyp_u = nullptr; // [n_utt] >= 1
  const float* lp_u = nullptr;    // [n_utt]
  // sampling (beam_size 1 with sampling_topk != 1; search.cu): every utterance keeps `beam` = num_hypotheses independent
  // rows, each sampling from softmax(l_S / temperature) with the Gumbel-max trick on a Philox stream keyed by the
  // utterance's seed.  best_len / best_score / best_tokens then hold one hypothesis per ROW ([R], [R], [R][max_new]);
  // max_hyp, n_cand and the per-utterance arrays are unused.
  int sample = 0;
  int topk = 0;                   // 0: every token with a finite processed logit; else in [2, MAX_CAND]
  float temperature = 1.f;        // finite, > 0
  const unsigned long long* seed_u = nullptr;  // [n_utt]
  // device word written by search_init: prompt positions a prefill pass forwarded into the cache slot of every window's
  // first row (0, prompt_len - 1, or prompt_len when that pass also produced the first step's logits, in its row
  // u * prompt_len + prompt_len - 1).  Positions below it are read from that slot by every row.  Null: 0.
  int* prompt_fed = nullptr;
};
void search_step_run(const SearchArgs& a, cudaStream_t stream);
// prompt prefill: no search, just feed the next prompt token and advance the position
void prefill_advance_run(int* tokens, const int* prompt /*[n_utt][prompt_len]*/, int prompt_len, int R, int beam,
                         DecState* st, cudaStream_t stream);
// fed: the prompt positions already in each window's prefix slot (SearchArgs::prompt_fed), 0 .. prompt_len; decoding
// starts at position min(fed, prompt_len - 1)
void search_init_run(const SearchArgs& a, const int* prompt, cudaStream_t stream, int fed = 0);
// rows of a batched prefill pass: row i = prompt position p0 + i % chunk of utterance i / chunk, cache slot = the
// utterance's first beam
void prefill_rows_run(int* tokens, int* row_pos, int* row_slot, const int* prompt, int prompt_len, int n_utt, int p0,
                      int chunk, int beam, cudaStream_t stream);

// ------------------------------------------------------------------ batched decoder pass (decoder_batch.cu)
struct BatchLayer {
  GemmPlan qkv, o, cq, co, fc1, fc2;  // built for the row capacity of the workspaces; o / co / fc2 write split-K partials
  const float *ln1g = nullptr, *ln1b = nullptr;      // LayerNorm before the QKV GEMM (only layer 0's is applied by the embedding kernel)
  const float *ob = nullptr, *ln2g = nullptr, *ln2b = nullptr;    // out-proj bias, LayerNorm before cross-attention
  const float *cob = nullptr, *ln3g = nullptr, *ln3b = nullptr;   // cross out-proj bias, LayerNorm before the MLP
  const float *fc2b = nullptr, *next_g = nullptr, *next_b = nullptr;  // fc2 bias, the NEXT LayerNorm (layer l+1's ln1 or the final one)
  const __half* ck = nullptr;   // cross K / V of this layer for utterance 0 of the pass: [n_utt][H][1536][64]
  const __half* cv = nullptr;
  __half* kcache = nullptr;     // self-attention cache of this layer: [slots][t_cap][d]
  __half* vcache = nullptr;
};
struct BatchArgs {
  int R = 0, d = 0, H = 0, n_utt = 0, rows_per_utt = 0, t_cap = 0, t_ind = 0, prefill = 0, with_logits = 0, pdl = 0;
  int wide = 0;                   // wide prefill pass: cross-attention through prefill_cross_attn_launch at any rows_per_utt
  const int* tokens = nullptr;    // [R]
  const int* row_pos = nullptr;   // [R]
  const int* row_slot = nullptr;  // [R]
  const __half* tok_emb = nullptr;
  const float* pos_emb = nullptr;
  float* x = nullptr;             // [rows_cap, d] fp32 residual stream
  __half* xn = nullptr;           // [rows_cap, d] LayerNorm output (GEMM A operand)
  float* q = nullptr;             // [rows_cap, d]
  __half* ctx = nullptr;          // [rows_cap, d] attention output (GEMM A operand)
  float* part = nullptr;          // split-K partial slabs [splits][rows_cap][d]
  long long part_stride = 0;
  const int* indir0 = nullptr;
  const int* indir1 = nullptr;
  const int* flip = nullptr;
  const int* done = nullptr;      // [n_utt] or null (prefill)
  const GemmPlan* vocab = nullptr;
  // wgmma cross-attention: one tensor map over the whole cross-K/V buffer viewed as [rows][64] fp16
  int cross_tc = 1, num_sms = 132;
  const CUtensorMap* ckv_map = nullptr;
  const __half* ckv_base = nullptr;
  // optional per-kernel-family timing hook (engine option "profile", eager launches only):
  // cat 0 GEMM, 1 cross-attention, 2 LayerNorm / embedding, 3 self-attention; begin = 1 / 0
  void (*prof)(void* ctx, int cat, int begin) = nullptr;
  void* prof_ctx = nullptr;
  // optional per-layer hook, called after the layer's cross-query GEMM (q holds the cross-attention queries); returns the
  // number of kernels it launched.  Null except in Whisper.align, which captures the alignment heads' attention there.
  int (*layer_hook)(void* ctx, int layer, cudaStream_t stream) = nullptr;
  void* hook_ctx = nullptr;
};
// returns the number of kernels launched
int batch_pass_run(const BatchArgs& a, const BatchLayer* layers, int n_layers, cudaStream_t stream);

// The launchers of the pass's own kernels.  batch_pass_run and the wisb_debug_dec_* entries (engine.cu) both launch
// through them; they check nothing but what the kernel choice depends on, so callers validate indices first.
// Utterances one cross-attention launch takes: the largest row capacity of a pass (option batch_rows) at one row each.
constexpr int BD_CROSS_MAX_UTT = 1024;
// x = tok_emb[tokens] + pos_emb[row_pos]; xn = LN(x) with gain g, shift b  (a.R rows of a.d <= 1536, a.d % 128 == 0)
void embed_ln_launch(const BatchArgs& a, const float* g, const float* b, cudaStream_t stream);
// ctx = self-attention of q over ly.kcache / ly.vcache through row_pos, row_slot, indir0 / indir1 (*flip), done, prefill
void self_attn_launch(const BatchArgs& a, const BatchLayer& ly, cudaStream_t stream);
// ctx = cross-attention of q over ly.ck / ly.cv; a.cross_tc picks the wgmma kernel (through a.ckv_map) or the SIMT one.
// More than 8 rows per utterance (prefill passes) always take prefill_cross_attn_launch.
void cross_attn_launch(const BatchArgs& a, const BatchLayer& ly, cudaStream_t stream);
// ctx = cross-attention of a.rows_per_utt (1..448) query rows per utterance, through a.ckv_map: the 128B-swizzled map over
// linear K/V, or a map without swizzle over the persistent pass's chunk-swizzled K/V (both give the same tile image)
void prefill_cross_attn_launch(const BatchArgs& a, const BatchLayer& ly, cudaStream_t stream);
// x += bias + the n_splits partial slabs at a.part (stride a.part_stride), in slab order; xn = LN(x)
void resid_ln_launch(const BatchArgs& a, int n_splits, const float* bias, const float* g, const float* b, cudaStream_t stream);

// ------------------------------------------------------------------ alignment (decoder_batch.cu, align.cu)
// Cross-attention probabilities of the alignment heads of one layer, captured during a teacher-forced batched prefill pass
// (rows_per_utt consecutive positions per utterance).  Item = (utterance, head of this layer).  P = softmax over all 1500
// keys of the fp16-rounded, 1/8-scaled query against the layer's cross K; written for positions s0 + r, 0 <= r <= n_text[u],
// frames f < n_frames[u] into cap [u][A][n_max + 1][f_max] at head index items[i].
struct AlignCaptureArgs {
  const float* q = nullptr;        // [n_utt * rows_per_utt, d] cross-attention queries (no scaling applied yet)
  const __half* ck = nullptr;      // cross K of this layer, utterance 0 of the pass: [n_utt][H][1536][64]
  const int* row_pos = nullptr;    // [rows] position of each row
  const int* items = nullptr;      // [n_items] global alignment-head index (into cap) of this layer's heads
  const int* head_of = nullptr;    // [A] head (within its layer) of every alignment head
  const int* n_text = nullptr;     // [n_utt]
  const int* n_frames = nullptr;   // [n_utt] F = num_frames // 2
  float* cap = nullptr;
  int n_items = 0, n_utt = 0, rows_per_utt = 0, d = 0, H = 0, A = 0, s0 = 0, n_max = 0, f_max = 0;
};
void align_capture_run(const AlignCaptureArgs& a, cudaStream_t stream);
// standardise cap over the rows (population std) per (utterance, head, frame), median-filter along frames (reflect
// padding, odd width <= 31; identity when F <= width / 2), mean over heads in head order -> mat [u][n_max + 1][f_max]
void align_filter_run(float* cap, float* mat, const int* n_text, const int* n_frames, int n_utt, int A, int n_max, int f_max,
                      int width, cudaStream_t stream);
// DTW on -mat per utterance (transformers _dynamic_time_warping, fp32 cost) -> path [u][path_stride][2] (text, time), len [u]
void align_dtw_run(const float* mat, const int* n_text, const int* n_frames, int n_utt, int n_max, int f_max, int* path,
                   int path_stride, int* path_len, cudaStream_t stream);
// text-token probabilities of one pass: for pass row (u, k) at position p = row_pos, i = p - s0 in [0, n_text[u]):
// probs[u][i] = softmax over ids [0, eot) of the row's logits, at text[u][i]
void align_token_probs_run(const float* logits, long long ldl, const int* row_pos, const int* text, int text_stride,
                           const int* n_text, int n_utt, int rows_per_utt, int s0, int eot, float* probs, cudaStream_t stream);

// ------------------------------------------------------------------ persistent decoder pass (decoder_mega.cu)
struct MegaGemv {
  const __half* w = nullptr;     // [N, K] fp16; K > 1536: chunk-major [chunk][N][K/chunks] (mega_chunk_major); warp-MMA pass: mega_mma_image
  const float* bias = nullptr;
  const float* ln_g = nullptr;   // LayerNorm gamma (x is multiplied by it while staged), K <= 1536
  const float* ln_s2 = nullptr;  // non-null = LayerNorm folded: s2[n] = sum_k g_k W[n,k]; `bias` then holds bias + sum_k b_k W[n,k]
  const float* x = nullptr;      // [R, K] fp32 activations
  float* out = nullptr;
  long long ldo = 0;
  int N = 0, K = 0, epi = GV_STORE;
  int shape = 0;                 // warp-MMA pass: 0 qkv, 1 d x d (o / cross-q / cross-o), 2 fc1, 3 fc2, 4 vocabulary (geometry table)
  // fp16 activation exchange images [K/64][R][64] (decoder_mega.cu act16_off): input read with one bulk copy / GELU output
  const __half* x16 = nullptr;
  __half* out16 = nullptr;
  const float* next_g = nullptr;  // GV_RESID: gain of the LayerNorm that reads the new residual rows next
};
struct MegaLayer {
  MegaGemv qkv, o, cq, co, fc1, fc2;
  const __half* ck = nullptr;    // cross K of this layer for the utterances of the pass: [n_utt][H][1536][64]
  const __half* cv = nullptr;
  __half* kcache = nullptr;      // self-attention cache of this layer: [slots][t_max][d]
  __half* vcache = nullptr;
};
struct MegaArgs {
  const MegaLayer* layers = nullptr;  // device array [n_layers]
  int n_layers = 0;
  MegaGemv vocab;
  int with_logits = 0;
  int R = 0, d = 0, H = 0, n_utt = 0, beam = 0, t_max = 0;
  // prompt prefill in one pass: rows = n_utt x pf_len prompt positions (beam := pf_len for the cross-attention phase),
  // tokens -> prompt [n_utt][pf_tok_stride], K/V written to cache slot u * pf_slot_stride; 0 = normal decoding step
  int pf_len = 0, pf_tok_stride = 0, pf_slot_stride = 0;
  const int* tokens = nullptr;
  const __half* tok_emb = nullptr;
  const float* pos_emb = nullptr;
  float* x = nullptr;      // [R, d] residual stream
  float* q = nullptr;      // [R, d]
  float* ctx = nullptr;    // [R, d]
  __half* ctx16 = nullptr; // warp-MMA pass: attention output as an fp16 exchange image instead of `ctx`
  __half* q16 = nullptr;   // warp-MMA pass: cross-attention queries [head][R][64] fp16, pre-scaled by 1/8
  __half* xn16 = nullptr;  // warp-MMA pass: residual rows times the next LayerNorm's gain, fp16 exchange image
  float* xstat = nullptr;  // warp-MMA pass: [CTA][R][2] per-CTA shares of the rows' (sum, sum of squares)
  const int* indir0 = nullptr;
  const int* indir1 = nullptr;
  const int* flip = nullptr;
  const DecState* st = nullptr;
  float* cross_part = nullptr;   // [n_utt][H][S<=16][MAX_BEAM][68] (64 acc, m, l, pad)
  unsigned* cross_flags = nullptr;  // [n_utt * H][16] epoch-tagged 'partial written' flags, one 128-byte line each
  unsigned* epoch_base = nullptr;  // [mega_flags_words()]: [0] epoch the last pass ended at, [8] grid-barrier counter
  int tc = 0;                    // 1: GEMV phases on the warp-level tensor path (dec_pass_mma_kernel)
};
size_t mega_flags_words();
int mega_k_chunks(int K);
void mega_chunk_major(const __half* src, __half* dst, int N, int K, cudaStream_t stream);
// W [N, K] -> the image the warp-MMA pass streams with one bulk copy per ring unit (N x K halves)
void mega_mma_image(const __half* src, __half* dst, int N, int K, int grid, cudaStream_t stream);
// s2[n] = sum_k g[k] W[n,k];  biasf[n] = bias[n] + sum_k b[k] W[n,k]   (bias may be null)
void mega_ln_fold(const __half* w, const float* g, const float* b, const float* bias, float* s2, float* biasf, int N, int K,
                  cudaStream_t stream);
void dec_pass_run(const MegaArgs& a, int num_sms, cudaStream_t stream);

// language detection head: softmax over lang ids of the logits of row u*beam (one step on <|startoftranscript|>)
void lang_probs_run(const float* logits, long long ldl, const int* lang_ids, int n_lang, int n_utt, int row_stride,
                    float* probs /*[n_utt][n_lang]*/, cudaStream_t stream);
// no-speech probability: out[u] = softmax over columns [0, n_vocab) of logits row rows[u], at column no_speech (raw
// logits: no suppression, processor or temperature).  Columns n_vocab .. ldl - 1 are never read.  rows[u] < 0: the
// window's row is not in this buffer and out[u] keeps its value.  One CTA per window, n_utt windows.
void no_speech_run(const float* logits, long long ldl, const int* rows /*[n_utt]*/, int n_utt, int n_vocab, int no_speech,
                   float* out /*[n_utt]*/, cudaStream_t stream);
// dst row u = src row rows[u] of d fp16 values (rows[u] < 0: dst row u keeps its value), u < n_utt
void row_gather_run(const __half* src, int d, const int* rows, int n_utt, __half* dst, cudaStream_t stream);

}  // namespace wisb
