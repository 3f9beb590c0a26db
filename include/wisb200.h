/* libwisb200 -- C ABI of the H100-native Whisper hot path that replaces, inside toverainc/willow-inference-server,
 *   (1) wis.audio.log_mel_spectrogram / pad_or_trim        (wis/audio.py:28-51, :72-103)
 *   (2) ctranslate2.models.Whisper(...)                     (main.py:341-355 and the four copies :363-443)
 *   (3) ctranslate2.StorageView.from_array(features)        (main.py:638, :685)
 *   (4) Whisper.generate(features, prompts, beam_size=...)  (main.py:687-692, positional form :535-537)
 *   (5) Whisper.detect_language(features)                   (main.py:638-640)
 *
 * Plain C: pointers and sizes only, no C++/torch types.  Every host buffer is owned by the caller and only borrowed for
 * the duration of the call; the handle owns device weights, workspaces, KV caches, streams and CUDA graphs.
 * All functions return 0 on success, 1 for invalid arguments (-> ValueError in the Python shim), 2 for CUDA/runtime
 * failures (-> RuntimeError); wisb_last_error() returns a thread-local message.  There is NO CPU fallback: without a
 * CUDA device every entry point except wisb_last_error / wisb_abi_version / wisb_generate_options_init fails with
 * code 2.
 * Calls on one handle are serialised internally; different handles may be used from different threads.
 */
#ifndef WISB200_H_
#define WISB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct wisb_handle wisb_handle;

#define WISB_ABI_VERSION 2
#define WISB_PCM_F32 0 /* float32 in [-1, 1]  (what librosa.load hands do_whisper, main.py:579) */
#define WISB_PCM_S16 1 /* int16 little endian (what /api/willow receives, main.py:1277-1299); scaled by 1/32768 on device */
#define WISB_N_DIMS 20

int wisb_abi_version(void);
const char* wisb_last_error(void);

/* (2) model construction.  `weights_path` is a WISB200 blob (willow_inference_server_b200/weights.py).  The *_host and
 * *_device forms take an in-memory blob; the device form borrows an already-populated device buffer (e.g. the target of
 * the load-time NCCL broadcast) which must outlive the handle. */
int wisb_create(const char* weights_path, int device, wisb_handle** out);
int wisb_create_from_host(const void* blob, size_t nbytes, int device, wisb_handle** out);
int wisb_create_from_device(const void* device_blob, size_t nbytes, int device, wisb_handle** out);
/* a handle without a model: only wisb_logmel works on it (wis.audio.log_mel_spectrogram is a free function).
 * wisb_create_frontend computes 80-bin features; wisb_create_frontend_mels takes the bin count, 80 or 128 (the
 * large-v3 family), and returns 1 for any other.  A model handle's front end has its model's n_mels. */
int wisb_create_frontend(int device, wisb_handle** out);
int wisb_create_frontend_mels(int device, int n_mels, wisb_handle** out);
int wisb_destroy(wisb_handle* h);
/* d_model, n_heads, n_enc_layers, n_dec_layers, n_vocab, n_vocab_pad, n_text_ctx, n_mels, n_audio_ctx, sot, eot,
 * transcribe, translate, no_timestamps, sot_prev, sot_lm, no_speech, blank, lang_first, n_langs */
int wisb_get_dims(wisb_handle* h, int32_t* dims /* [WISB_N_DIMS] */);

/* (1) batched log-mel.  Utterance b is n_samples[b] samples starting at pcm + offsets[b] (in samples); padding with
 * zeros / trimming to 480000 samples is fused.  pcm_on_device != 0: `pcm` is a device pointer.  n_mels below is the
 * handle's (wisb_get_dims entry 7): 80, or 128 for the large-v3 family; a blob with any other value is refused (code 1).
 * mel_out (host, float32 [B,n_mels,3000]) may be NULL; keep_on_device != 0 keeps the features in HBM for the next
 * wisb_generate / wisb_detect_language call that passes mel == NULL. */
int wisb_logmel(wisb_handle* h, const void* pcm, int pcm_dtype, int pcm_on_device, const int64_t* offsets,
                const int32_t* n_samples, int B, float* mel_out, int keep_on_device);

/* (4) the options of Whisper.generate (main.py:687-692), CTranslate2's defaults from wisb_generate_options_init.
 * struct_size is sizeof(wisb_generate_options) as the caller was compiled (wisb_generate refuses any other value).
 * Every per-window array is [B] or NULL, NULL meaning "the scalar applies to every window". */
typedef struct wisb_generate_options {
  uint32_t struct_size;
  /* beam search (sampling_topk == 1): beam_size in [1, 8], 1 = greedy.  A window finishes once max(1, round half up of
   * beam_size x patience in fp32) hypotheses exist (patience finite, > 0) and ranks them by cumulative log-prob over
   * (generated tokens)^length_penalty (finite). */
  int32_t beam_size;            /* 5 */
  float patience;               /* 1 */
  float length_penalty;         /* 1 */
  /* at most min(max_length / 2, max_length - prompt_len) new tokens; max_length in [1, n_text_ctx] */
  int32_t max_length;           /* 448 */
  /* Whisper's timestamp rules, 0 or 1: what CTranslate2 does for a prompt WITHOUT <|notimestamps|> (the 3-token sot,
   * language, task prompt).  The returned ids then contain timestamp tokens (ids > no_timestamps), which come in pairs
   * except directly before <|endoftext|> and never decrease; the first generated token is a timestamp <= no_timestamps
   * + 1 + max_initial_timestamp_index (50: 1.00 s).  The rules read only the generated tokens, so with timestamps the
   * prompt may hold any ids, timestamps included, BEFORE its last <|startoftranscript|> (a <|startofprev|> context of
   * earlier windows' output, as faster-whisper builds with condition_on_previous_text, initial_prompt or hotwords);
   * from that <|startoftranscript|> on (the whole prompt when it has none) it must contain neither <|notimestamps|> nor
   * timestamp tokens.  transformers applies its rules from the same begin index; CTranslate2's own check on such prompts
   * is UNPINNED.  max_initial_timestamp_index >= 0 in both modes. */
  int32_t timestamps;                   /* 0 */
  int32_t max_initial_timestamp_index;  /* 50 */
  /* the history processors: repetition_penalty (finite, > 0; 1 = off) divides a positive logit and multiplies a
   * negative one of every distinct token the hypothesis has generated so far; no_repeat_ngram_size (in [0, n_text_ctx];
   * 0 = off) bans every token that would complete an n-gram the hypothesis already holds.  History = the hypothesis's
   * generated tokens (timestamp tokens included, prompt tokens not).  They apply before the suppress masks and the
   * timestamp rules. */
  float repetition_penalty;      /* 1 */
  int32_t no_repeat_ngram_size;  /* 0 */
  /* sampling_topk != 1 samples (CTranslate2's rule; beam_size must then be 1, patience is not read and no per-window
   * search option may be given): every window draws num_hypotheses (in [1, 8]; 1 unless sampling) independent
   * hypotheses from softmax(l_S / sampling_temperature) (finite, > 0) over the processed logits l, S = every token
   * (sampling_topk 0) or the sampling_topk (in [2, 16]) largest, with Gumbel-max noise from Philox4x32-10 keyed by
   * seeds[b].  The result depends only on the window's features, prompt, options and seed, not on its batch position.
   * Scores are the untempered cumulative log-probs over (generated tokens)^length_penalty. */
  int32_t num_hypotheses;        /* 1 */
  int32_t sampling_topk;         /* 1 */
  float sampling_temperature;    /* 1 */
  /* ids suppressed in addition to the model's suppress_ids (CT2 `suppress_tokens=[-1, ...]`) */
  int32_t n_extra;
  const int32_t* extra_suppress;
  /* The per-window options are what CTranslate2's per-call options become when a batcher coalesces several calls into
   * ONE shared decoder pass.  max_length_per_window in [1, n_text_ctx].  beam_per_window in [1, 8],
   * patience_per_window finite and > 0, length_penalty_per_window finite: window b searches with its own beam, patience
   * and length penalty exactly as it would alone.  Every window keeps a block of rows of the largest beam B of its group
   * (at most batch_rows / B windows per group), searches its first b rows and leaves the others dead; a group whose
   * windows agree on beam, max_hyp and length penalty runs the scalar search. */
  const int32_t* max_length_per_window;
  const int32_t* beam_per_window;
  const float* patience_per_window;
  const float* length_penalty_per_window;
  const uint64_t* seeds;  /* uint64 [B], required when sampling */
} wisb_generate_options;

/* CTranslate2's defaults (the values above, every pointer NULL) and struct_size; needs no CUDA device and no handle.
 * Code 1 if opt is NULL. */
int wisb_generate_options_init(wisb_generate_options* opt);

/* (3)+(4) features [B,n_mels,3000] float32 host (or NULL: use the features kept by wisb_logmel) -> token ids.
 * prompts: int32 [B, prompt_len] (WIS passes the same 4-token prompt for every window, main.py:689).
 * Outputs hold n = num_hypotheses entries per window when sampling, else one: window b's at [b * n, (b + 1) * n),
 * sorted by score (descending, ties to the lower hypothesis index).  out_ids int32 [B * n, out_stride] (out_stride >=
 * the largest number of new tokens of any window), out_len int32 [B * n], out_score float32 [B * n] (may be NULL unless
 * sampling) the length-normalised log-probability of each hypothesis.  A sampled hypothesis that found no token to
 * sample is empty with score -inf; a cap of 0 new tokens gives n empty ones with score 0.  Code 1 for a bad argument. */
int wisb_generate(wisb_handle* h, const float* mel, int B, const int32_t* prompts, int prompt_len,
                  const wisb_generate_options* opt, int32_t* out_ids, int out_stride, int32_t* out_len, float* out_score);

/* (5) per utterance: language token ids sorted by probability (descending) and the probabilities.
 * lang_ids_out int32 [B, n_langs], probs_out float32 [B, n_langs]. */
int wisb_detect_language(wisb_handle* h, const float* mel, int B, int32_t* lang_ids_out, float* probs_out);

/* (5b) Whisper.align: token-to-frame alignment from the cross-attention of the alignment heads (blob tensor
 * meta.alignment_heads [A, 2] (layer, head); without it every head of layers n_dec_layers / 2 .. n_dec_layers - 1).
 * mel as in wisb_generate (NULL = the features wisb_logmel kept on the device).  Window b is teacher-forced with
 * start_seq [start_len] + <|notimestamps|> + text[b, :text_len[b]]; start_seq begins with <|startoftranscript|> and holds
 * neither <|notimestamps|> nor timestamp ids, text ids are in [0, eot), start_len + 1 + text_len[b] <= n_text_ctx,
 * num_frames[b] in [2, 3000], median_filter_width odd in [1, 31], path_stride >= text_len[b] + num_frames[b] / 2 + 1 (the longest path: R + F
 * entries, reached when NaN columns of the filtered matrix, frames whose probabilities are equal in every row, route it
 * along the last row to frame 0).
 * Outputs: out_path int32 [B, path_stride, 2] = (text index in [0, text_len], frame in [0, num_frames / 2)) in path order,
 * out_path_len [B], out_token_probs float32 [B, text_stride] (entry i < text_len[b]: probability of text token i).
 * A window with text_len 0 gets an empty path and adds no capture, filter or DTW work.  Stage timings in wisb_get_timing:
 * [1 h2d, 2 encoder + cross K/V, 3 teacher-forced passes (capture and token probabilities included), 4 filter, 5 total,
 *  6 passes, 7 kernel launches, 13 capture kernels (option "profile" only), 14 DTW]. */
int wisb_align(wisb_handle* h, const float* mel, int B, const int32_t* start_seq, int start_len, const int32_t* text,
               const int32_t* text_len, int text_stride, const int32_t* num_frames, int median_filter_width,
               int32_t* out_path, int path_stride, int32_t* out_path_len, float* out_token_probs);

/* (7) encoder output as a value of its own, CTranslate2's Whisper.encode: faster-whisper encodes each window once and
 * passes the result to detect_language, to generate (once per temperature retry) and to align.
 * wisb_buffer_alloc: `nbytes` of device memory on `device`, owned by no handle (the library links the CUDA runtime
 * statically, so a caller has no other way to allocate device memory it can hand back here).  wisb_buffer_free works from
 * any current device and after every handle is destroyed; NULL is a no-op, any other pointer it did not hand out is
 * refused (code 1). */
int wisb_buffer_alloc(int device, size_t nbytes, void** out);
int wisb_buffer_free(void* p);
/* the first nbytes (<= its size) of a live wisb_buffer_alloc buffer -> host memory; blocks until the copy is done */
int wisb_buffer_to_host(const void* p, void* host, size_t nbytes);
/* features [B,n_mels,3000] float32 host (or NULL: the features kept by wisb_logmel) -> the encoder output after the final
 * LayerNorm, fp16 [B, 1500, d_model], into `out`: a host pointer, or (out_on_device != 0) device memory on the handle's
 * device.  Encodes in groups of at most option batch_rows / 5 windows (generate's group at beam 5), so it sizes no
 * workspace beyond what generate would.  Invalidates the cached encoder output.  Stage timings: [1 h2d, 2 encoder,
 * 5 total, 7 kernel launches] and, with option "profile", 8-12 as for generate. */
int wisb_encode(wisb_handle* h, const float* mel, int B, void* out, int out_on_device);
/* An encoder output [B, 1500, d_model] (dtype 0 fp16, 1 fp32: converted on the device, rounded to nearest even), host
 * memory or (on_device != 0) device memory on the handle's device, copied into a handle-owned buffer.  It becomes the
 * source of the next wisb_generate / wisb_detect_language / wisb_align calls that pass mel == NULL: whichever of
 * wisb_logmel(keep_on_device) and this call came last decides that source, and such a call with another B fails with
 * code 1.  Those calls skip the encoder and run only the cross-K/V GEMM on these rows; they leave nothing for option
 * "encoder_cache" to reuse.  A host copy's time is reported in timing slot 1 (h2d). */
int wisb_load_encoder_output(wisb_handle* h, const void* enc, int B, int dtype, int on_device);

/* stage timings (ms, CUDA events on the launching stream) of the last wisb_logmel / wisb_generate:
 * [0 logmel, 1 h2d, 2 encoder, 3 cross_kv, 4 decode, 5 total_generate, 6 decode_steps, 7 kernel_launches,
 *  8 sum of GEMM kernels, 9 attention kernels, 10 LayerNorm kernels, 11 conv1, 12 number of GEMM launches, 13-15 0]
 * entries 8-12 are filled only with option "profile" = 1 (per-kernel event pairs; leave it off for timed runs). */
int wisb_get_timing(wisb_handle* h, float* out16);
/* options: "use_graphs" (default 1), "attn_v_mn_major" (default 1), "attn_ref" (0), "profile" (0),
 * "mega_mma" (for calls of <= 8 rows: 1, the default where d_model <= 1280, the warp-MMA persistent decoder pass; 0 the
 * SIMT persistent pass, fp32 arithmetic, the only one for d_model > 1280),
 * "encoder_cache" (default 0; 1: consecutive wisb_detect_language / wisb_generate / wisb_align calls on byte-identical
 * host features of <= 2 windows reuse the encoder output and cross K/V already in HBM when the call encodes all its
 * windows in one group -- the detect -> transcribe -> translate sequence of main.py:633-644, 514-547 then encodes once
 * instead of three times; cached cross K/V in the other decoder pass's layout is rewritten by the cross-K/V GEMM alone),
 * "wide_prefill" (default 1; 0: prompts prefill at most 8 positions per pass, one persistent pass per position when the
 * one-pass prefill does not fit), "prefill_rows" (default 1024, 8..65536: a prompt of more than 9 tokens is prefilled in
 * batched passes of min(prompt_len - 1, max(the 8-position chunk, prefill_rows / windows)) positions per window; it
 * bounds the prefill's activation workspace, about 52 d_model bytes per row),
 * "no_speech_prob" (default 0; 1: every wisb_generate also computes each window's no-speech probability, read with
 * wisb_get_no_speech_probs) */
int wisb_set_option(wisb_handle* h, const char* key, int value);

/* (4b) The no-speech probabilities of the handle's last wisb_generate, one per window (also when sampling), into out
 * float32 [B].  Window b's value is softmax(l)[no_speech] of the decoder's raw logits l over the whole vocabulary at
 * the position of the FIRST <|startoftranscript|> in its prompt (openai/whisper's sot_index), before suppression,
 * history processors, timestamp rules and temperature; a window capped at 0 new tokens gets its value too.  With option
 * "no_speech_prob" = 1, wisb_generate fails with code 1 for a prompt without <|startoftranscript|>, and its ids, lengths,
 * scores and decoder passes are those of the same call without the option.  Code 1 when that call ran without the
 * option, failed, or had another B. */
int wisb_get_no_speech_probs(wisb_handle* h, int B, float* out);

/* ---- diagnostics used by tests/ (run the product kernels on caller data) ---- */
/* One GEMM A[M,K] . W[N,K]^T (fp16 as raw uint16) through any production epilogue, on caller data.
 * prm[17] int32: M, N, K, impl (0 = wgmma kernel, 1 = SIMT check into float32 out [M,N]), bn (0 = encoder planner's
 * choice, 64/128/160/256, negative = that width without 2-CTA multicast), planner (0 = encoder planner, 1 = decoder
 * planner, 2 = decoder planner with split-K: float32 partial slabs of M*N), mode (EpiMode of csrc/kernels.h), a_wrap
 * (> 0: A is given as its physical [M+1, a_wrap] rows, the overlapping-row view of conv2), k_splits (> 1: float32 slabs
 * of M*ldo), m_valid, n_valid (0 = M, N), ldo (0 = N), d_model, n_heads, batch, kv_swizzle, t_cap.
 * bias [N] and pos [1500, ldo] may be NULL; row_slot / row_pos [M] are the cache slot / position of each row (DEC_QKV).
 * out / aux / aux2 are uploaded before the launch and downloaded after it, so that untouched elements keep what the
 * caller put there; every address the epilogue can form is checked against their byte sizes first.
 * plan_out (may be NULL) receives the launched plan: BN, multicast (0/1), K splits, grid. */
int wisb_debug_gemm(wisb_handle* h, const int32_t* prm, int n_prm, const uint16_t* a, const uint16_t* w, const float* bias,
                    const float* pos, const int32_t* row_slot, const int32_t* row_pos, void* out, size_t out_bytes, void* aux,
                    size_t aux_bytes, void* aux2, size_t aux2_bytes, int32_t* plan_out);
/* ONE production token-search step (wisb_generate's processors, top-k or sampling, bookkeeping and step advance) on
 * caller search state, which it returns.  prm[15] int32: n_utt, beam, V, ldl (>= V), eot, no_timestamps, timestamps
 * (0/1), max_initial_timestamp_index, max_new (1..448), max_hyp (>= 1), t_max (1..448), init (0: the state as given;
 * 1 / 2: search initialisation from `prompt` first, with shared_prefix 0 / 1), prompt_len, no_repeat_ngram_size,
 * sampling_topk (1 = search).  fprm[3] float32: length_penalty, repetition_penalty, sampling_temperature.  The options
 * mean what they mean in wisb_generate_options.  n_utt * beam <= 1024.
 * logits float32 [n_utt*beam, ldl] (columns >= V are never read); mask uint8 [V] (bit 0: suppressed every step, bit 1:
 * at the first generated step); max_new_u int32 [n_utt] per-utterance caps in [0, max_new] or NULL; prompt int32
 * [n_utt, prompt_len] (init only).  state_i int32 in / out: DecState {pos, gen_step, n_done, all_done, ticket (0)},
 * flip, seq [2][R][max_new], indir [2][R][t_max], tokens [R], row_pos [R], done [n_utt], n_hyp [n_utt], best_len
 * [H], best_tokens [H][max_new]; state_f float32 in / out: cum [R], best_score [H]  (R = n_utt * beam; H = n_utt, or R
 * when sampling: one hypothesis per row).
 * Per-utterance search options (beam_u, max_hyp_u, length_penalty_u: all three, or none) make prm[1] the row block B of
 * every utterance: utterance u searches rows [0, beam_u[u]) (beam_u[u] in [1, B]) with 2 beam_u[u] candidates,
 * finishes at max_hyp_u[u] (>= 1) hypotheses and normalises with length_penalty_u[u] (finite); prm[9] (>= 1) and
 * fprm[0] are unused.  Its other rows are dead: cum -inf, token eot, never a candidate (cand_idx entries 2 beam_u[u] ..
 * 15 are -1) or a hypothesis.  With init, search initialisation makes them dead.  Sampling takes none of them; prm[1]
 * is then the hypotheses n per utterance, prm[9] (>= 1) is unused and seeds is uint64 [n_utt].
 * Outputs: cand_idx int32 [n_utt, 16] and cand_score float32 [n_utt, 16]: searching, the first 2*beam entries are the
 * candidates (beam * V + token, -1 = none) and their scores; sampling, entry k < n is the token row k drew (-1 = none:
 * the row was dead, frozen or had nothing to sample) and its Gumbel key.  row_lse float32 [n_utt*beam].  Sizes, the
 * current history tokens and indirection entries are checked before anything is launched. */
int wisb_debug_search_step(wisb_handle* h, const int32_t* prm, int n_prm, const float* fprm, int n_fprm,
                           const float* logits, const uint8_t* mask, const int32_t* max_new_u, const int32_t* prompt,
                           const int32_t* beam_u, const int32_t* max_hyp_u, const float* length_penalty_u,
                           const uint64_t* seeds, int32_t* state_i, float* state_f, int32_t* cand_idx, float* cand_score,
                           float* row_lse);
/* the no-speech reduction on caller data: out[u] = softmax over columns [0, n_vocab) of row rows[u] of logits float32
 * [n_rows, ldl], at column no_speech (columns >= n_vocab are never read).  rows[u] < 0 leaves out[u] as the caller gave
 * it.  n in [1, 65535], n_vocab <= ldl, rows[u] < n_rows. */
int wisb_debug_no_speech_probs(wisb_handle* h, const float* logits, int n_rows, int ldl, const int32_t* rows, int n,
                               int n_vocab, int no_speech, float* out);
/* encoder self-attention on caller data: qkv [B*1536, 3d] fp16 -> ctx [B*1536, d] fp16, d = 64 H; impl 0 = wgmma with
 * MN-major V, 1 = wgmma with the transposed Vt layout (built from the same qkv), 2 = SIMT check */
int wisb_debug_enc_attn(wisb_handle* h, const uint16_t* qkv16, int B, int d, int H, int impl, uint16_t* ctx16_out);
/* The batched decoder pass's own kernels on caller data, launched exactly as the pass launches them (without
 * programmatic dependent launch).  fp16 arrays are raw uint16.  Outputs are uploaded before the launch and downloaded
 * after it, so elements the kernel must not write keep what the caller put there.  Every index a kernel can form is
 * checked against the sizes given here first: a bad argument returns 1 and launches nothing. */
/* cross-attention.  prm[6] int32: n_utt (1..1024), rows_per_utt (1..8), H (1..32), n_layers, layer, impl (0 = wgmma
 * kernel through a tensor map over the whole buffer, 1 = SIMT cluster kernel).  d = 64 H.  q float32 [n_utt *
 * rows_per_utt, d] (unscaled), ckv [n_layers][2 (K, V)][n_utt][H][1536][64] (keys >= 1500 are padding), done int32
 * [n_utt] or NULL (finished utterances are skipped), ctx [n_utt * rows_per_utt, d] in / out. */
int wisb_debug_dec_cross_attn(wisb_handle* h, const int32_t* prm, int n_prm, const float* q, const uint16_t* ckv,
                              const int32_t* done, uint16_t* ctx16);
/* self-attention over a beam-indirected cache.  prm[8] int32: R, H (1..32), n_slots, t_cap, t_ind (<= 448),
 * rows_per_utt (1..8, divides R), prefill (0/1), flip (0/1: which indirection table is current).  d = 64 H.  q float32
 * [R, d], kcache / vcache [n_slots][t_cap][d], row_pos / row_slot int32 [R] (row_pos < min(t_cap, t_ind)), indir0 /
 * indir1 int32 [R][t_ind] (slots), done int32 [R / rows_per_utt] or NULL, ctx [R, d] in / out.  Row r attends positions
 * t <= row_pos[r]: slot indir[r][t] for t < row_pos[r], its own slot row_slot[r] at t = row_pos[r] (and at every t with
 * prefill). */
/* cross-attention of a wide prefill pass (more than 8 query rows per utterance), the kernel the engine's prefill passes
 * launch.  prm[6] int32: n_utt (1..1024), rows_per_utt (1..448), H (1..32), n_layers, layer, swizzled (0: ckv in the
 * linear layout of the batched pass, 1: in the persistent warp-MMA pass's layout, where 16-byte chunk c of key t's
 * 128-byte row lies at chunk c ^ (t & 7)).  d = 64 H.  q float32 [n_utt * rows_per_utt, d] (unscaled), ckv
 * [n_layers][2 (K, V)][n_utt][H][1536][64] (keys >= 1500 are padding and may hold anything), ctx [n_utt * rows_per_utt,
 * d] in / out. */
int wisb_debug_dec_prefill_cross_attn(wisb_handle* h, const int32_t* prm, int n_prm, const float* q, const uint16_t* ckv,
                                      uint16_t* ctx16);
int wisb_debug_dec_self_attn(wisb_handle* h, const int32_t* prm, int n_prm, const float* q, const uint16_t* kcache,
                             const uint16_t* vcache, const int32_t* row_pos, const int32_t* row_slot, const int32_t* indir0,
                             const int32_t* indir1, const int32_t* done, uint16_t* ctx16);
/* split-K reduction + bias + residual + LayerNorm: x[r] += ((bias + slab 0) + slab 1) + ..., xn = LN(x) (fp16).
 * d % 128 == 0, d <= 1536; n_splits 1, 2, 4 or 8 slabs of [R, d] float32 at part + s * split_stride (split_stride % 4
 * == 0, >= R d when n_splits > 1, part_elems >= (n_splits - 1) split_stride + R d); bias, g, b float32 [d]; x float32
 * [cap, d] and xn [cap, d] in / out (cap >= R: rows R .. cap - 1 must come back untouched). */
int wisb_debug_dec_resid_ln(wisb_handle* h, int R, int cap, int d, int n_splits, int64_t split_stride, const float* part,
                            size_t part_elems, const float* bias, const float* g, const float* b, float* x, uint16_t* xn16);
/* token + position embedding + LayerNorm: x[r] = float(tok_emb[tokens[r]]) + pos_emb[row_pos[r]], xn = LN(x).  tok_emb
 * [n_vocab, d] fp16, pos_emb [n_pos, d] float32, g, b float32 [d]; x float32 [cap, d] and xn [cap, d] in / out (cap >= R). */
int wisb_debug_dec_embed_ln(wisb_handle* h, int R, int cap, int d, int n_vocab, int n_pos, const int32_t* tokens, const int32_t* row_pos,
                            const uint16_t* tok_emb, const float* pos_emb, const float* g, const float* b, float* x,
                            uint16_t* xn16);
/* ONE persistent decoder pass on caller state, launched exactly as decoding launches it.  prm = {impl (1 warp-MMA,
 * 0 SIMT), n_utt, beam, pf_len, pos, flip, with_logits}.  Decoding step (pf_len 0): R = n_utt * beam <= 8 rows at
 * position pos (0..447), tokens[R], cache indirection indir0 / indir1 int32 [R][448] (flip picks indir1).  One-pass
 * prompt prefill (pf_len >= 1): R = n_utt * pf_len <= 8 rows, row u * pf_len + p = prompt position p of utterance u,
 * written to cache slot u * beam; pos, flip and indir are unused.  enc16: fp16 encoder rows [n_utt][1536][d] (padding
 * rows included) -> the cross K/V through the cross-K/V GEMM; ckv_out receives it in the plain layout, [L][2][n_utt][H]
 * [1536][64] fp16.  kcache / vcache: fp16 [L][8][448][d] in / out; x: float32 [8][d] in / out (rows < R are the
 * pass's residual stream); logits: float32 [8][n_vocab_pad] in / out (rows < R, columns < n_vocab written when
 * with_logits).  Invalidates the cached encoder output. */
int wisb_debug_dec_pass(wisb_handle* h, const int32_t* prm, int n_prm, const int32_t* tokens, const int32_t* indir0,
                        const int32_t* indir1, const uint16_t* enc16, uint16_t* ckv_out, uint16_t* kcache, uint16_t* vcache,
                        float* x, float* logits);
/* ONE batched decoder pass on caller state, with the workspaces, GEMM plans, row tables and arguments of its production
 * caller.  prm (16) = {kind, n_utt, rows_per_utt, slot_stride, prompt_len, p0, batch_rows, t_need, chunk_max, flip,
 * with_logits, cross_tc, ckv_sw, poison, poison_slot, poison_pos}.
 *   kind 0  decoding step: R = n_utt * rows_per_utt (<= 8 per window) rows, row r at row_pos[r] in cache slot r, tokens[R],
 *           indir0 / indir1 int32 [R][448] (flip picks indir1) for the positions below row_pos[r], done int32 [n_utt] or
 *           NULL; with_logits 1; cross_tc picks the wgmma (1) or SIMT (0) cross-attention
 *   kind 1  batched prefill: positions p0 .. p0 + rows_per_utt - 1 (<= 8) of every window of the prompt matrix tokens
 *           [n_utt][prompt_len] as rows u * rows_per_utt + i, K/V into slot u * slot_stride; with_logits 0 / 1
 *   kind 2  wide prefill pass (rows_per_utt <= chunk_max <= 448 positions per window) into the batched cache
 *   kind 3  wide prefill pass into the persistent pass's cache; ckv_sw: the cross K/V are in its chunk-swizzled layout
 * Kinds 0..2 size the batched workspaces for batch_rows rows and t_need positions (they only grow within a handle); wide
 * passes size their own for n_utt * chunk_max rows.  ckv: fp16 [L][2][n_utt][H][1536][64] in the layout the pass reads.
 * geom_out int64 [4] <- cache slots, positions per slot (t_cap), layer stride in elements, row capacity of the
 * workspaces; kcache / vcache fp16 [L][slots][t_cap][d] in / out; x float32 [R][d] out; logits float32 [R][n_vocab_pad]
 * out in columns < n_vocab (the others keep the caller's values).  kcache NULL: the geometry only, nothing allocated or
 * launched.  plan_out (may be NULL) int32 [7][4]: BN, multicast, K splits and grid of the qkv, o, cq, co, fc1, fc2 and
 * vocabulary GEMMs (vocabulary 0 in wide passes).
 * poison 1: rows >= R of every activation workspace and partial slab hold NaN during the pass (restored after), row-
 * table entries >= R point at cache cell (poison_slot, poison_pos), which the pass must not write.  Every index
 * (tokens, positions < min(t_cap, n_text_ctx), slots, indirection entries, rows) is checked against that geometry
 * before any workspace is sized or anything launched; a refused call returns 1 and changes nothing.  Invalidates the
 * cached encoder output. */
int wisb_debug_dec_batch_pass(wisb_handle* h, const int32_t* prm, int n_prm, const int32_t* tokens, const int32_t* row_pos,
                              const int32_t* indir0, const int32_t* indir1, const int32_t* done, const uint16_t* ckv,
                              uint16_t* kcache, uint16_t* vcache, float* x, float* logits, int64_t* geom_out, int32_t* plan_out);
/* encoder output after the final LayerNorm, float32 [B,1500,d_model]; n_layers < 0 = all */
int wisb_debug_encode(wisb_handle* h, const float* mel, int B, float* enc_out, int n_layers);
/* The encoder one stage at a time, through the functions the encoder itself runs.  Sizes and indices are checked before
 * anything is launched (a bad argument returns 1); each entry invalidates the cached encoder output.  fp16 as raw uint16.
 * stem: conv1 + the conv2 GEMM on log-mel float32 [B,n_mels,3000] (1 <= B <= 4096) -> h1_out fp16 [B * 3072 + 8, d] (conv1
 * output, all of it: window b's frame f at row b * 3072 + 1 + f, zero rows 0 and 3001..3071 of each window, 8 tail rows)
 * and x_out float32 [B * 1536, d] (conv2 + positions; rows 1500..1535 of each window are padding). */
int wisb_debug_enc_stem(wisb_handle* h, const float* mel, int B, uint16_t* h1_out, float* x_out);
/* the encoder LayerNorm on caller data: x float32 [rows, d] (d a multiple of 128, <= 1536), g, b float32 [d], pdl 0 / 1
 * (launch with programmatic dependent launch) -> y fp16 [round_up(rows, 8), d] in / out: rows >= `rows` of the kernel's
 * last 8-row block come back as the caller put them. */
int wisb_debug_enc_ln(wisb_handle* h, const float* x, int rows, int d, const float* g, const float* b, int pdl, uint16_t* y);
/* the seven launches of encoder layer `layer` on the residual x_in float32 [B * 1536, d] (padding rows included) ->
 * x_out float32 [B * 1536, d].  stages_out (may be NULL) receives the output of every launch, at byte offsets in units
 * of md = B * 1536 * d: 0 xn1 fp16 [md], 2 qkv fp16 [B * 1536, 3 d], 8 vt fp16 [B, H, 64, 1536] (as the QKV epilogue
 * leaves it: written only under attn_v_mn_major = 0, when qkv's V columns are not), 10 ctx fp16 [md], 12 x after the
 * o-projection float32 [md], 16 xn2 fp16 [md], 18 fc1 output fp16 [B * 1536, 4 d]; 26 md bytes in all.  Taking the
 * snapshots serialises the chain; without them it runs as the encoder does (options enc_pdl, attn_v_mn_major, attn_ref).
 * plan_out (may be NULL) int32 [4][4]: BN, multicast, K splits and grid of the qkv, o, fc1 and fc2 GEMMs. */
int wisb_debug_enc_layer(wisb_handle* h, int layer, int B, const float* x_in, float* x_out, void* stages_out, int32_t* plan_out);
/* teacher-forced raw decoder logits (no processors) for utterance 0: float32 [n_tokens, n_vocab] */
int wisb_debug_forced_logits(wisb_handle* h, const float* mel, const int32_t* tokens, int n_tokens, float* logits_out);
/* wisb_align's post-processing kernels on caller data for one window: weights float32 [A, R, F] (R = text rows + 1,
 * 2 <= R <= 449, 1 <= F <= 1500) -> standardise, median filter of odd `width` <= 31, head mean -> matrix_out float32
 * [R, F] (may be NULL), then DTW -> path_out int32 [R + F, 2], path_len.  dtw_only = 1: weights is the matrix [R, F]
 * itself (A = 1) and only the DTW runs. */
/* wisb_align's teacher-forced passes on caller data, returning the raw captured probabilities (before the filter):
 * cap_out float32 [B, A, n_max + 1, F_max] with n_max / F_max the largest text_len / num_frames / 2 over the windows that
 * have text; entry [b, a, r, f] (r <= text_len[b], f < num_frames[b] / 2) is alignment head a's softmax over all 1500
 * frames at row r, other entries are left as they were.  The windows must fit in one group of wisb_align. */
int wisb_debug_align_capture(wisb_handle* h, const float* mel, int B, const int32_t* start_seq, int start_len,
                             const int32_t* text, const int32_t* text_len, int text_stride, const int32_t* num_frames,
                             float* cap_out);
int wisb_debug_align_post(wisb_handle* h, const float* weights, int A, int R, int F, int width, int dtw_only,
                          float* matrix_out, int32_t* path_out, int32_t* path_len);

/* ---- (6) FLAC ingest (host code, no handle, no GPU): replaces the decode half of `librosa.load(audio_file, sr=16000)`
 * (main.py:579) for the FLAC files WIS is tested with (client/{3sec,10sec,30sec}.flac).
 * wisb_flac_info: stream parameters, number of inter-channel frames and the PCM MD5 from STREAMINFO (any pointer may be NULL).
 * wisb_flac_decode: interleaved int32 samples [n_frames, channels]; every frame's CRC-8 / CRC-16 is checked.
 * Both return 0 or a non-zero code with the reason in wisb_flac_last_error() (thread-local). */
const char* wisb_flac_last_error(void);
int wisb_flac_info(const void* data, size_t nbytes, int32_t* sample_rate, int32_t* channels, int32_t* bits_per_sample,
                   int64_t* n_frames, uint8_t* md5_16);
int wisb_flac_decode(const void* data, size_t nbytes, int32_t* out_interleaved, int64_t capacity_frames, int64_t* n_frames);

#ifdef __cplusplus
}
#endif
#endif /* WISB200_H_ */
