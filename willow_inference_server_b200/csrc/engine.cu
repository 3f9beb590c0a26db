// libwisb200.so host side: handle, weight blob, workspaces, encoder / decoder orchestration and the C ABI
// declared in include/wisb200.h.  Mirrors the call surface WIS uses on ctranslate2 (main.py:341-355, 638-640, 685-692).
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/wisb200.h"
#include "decoder.cuh"
#include "kernels.h"

namespace wisb {

namespace {

thread_local std::string g_last_error;

struct TensorRef {
  const uint8_t* ptr = nullptr;
  int dtype = 0, ndim = 0;
  long long shape[4] = {1, 1, 1, 1};
  long long numel() const { return shape[0] * shape[1] * shape[2] * shape[3]; }
};

struct Dims {
  int d_model, n_heads, n_enc_layers, n_dec_layers, n_vocab, n_vocab_pad, n_text_ctx, n_mels, n_audio_ctx, sot, eot,
      transcribe, translate, no_timestamps, sot_prev, sot_lm, no_speech, blank, lang_first, n_langs;
};
static_assert(sizeof(Dims) == WISB_N_DIMS * sizeof(int), "Dims must mirror the blob header");

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  void ensure(size_t count, bool zero = false) {
    if (count <= n) return;
    release();
    WISB_CUDA(cudaMalloc(&p, count * sizeof(T)));
    n = count;
    if (zero) WISB_CUDA(cudaMemset(p, 0, count * sizeof(T)));
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  ~DevBuf() { release(); }
};

template <typename T>
struct PinBuf {
  T* p = nullptr;
  size_t n = 0;
  void ensure(size_t count) {
    if (count <= n) return;
    if (p) cudaFreeHost(p);
    WISB_CUDA(cudaMallocHost(&p, count * sizeof(T)));
    n = count;
  }
  ~PinBuf() {
    if (p) cudaFreeHost(p);
  }
};

struct EncLayerPlans {
  GemmPlan qkv, o, fc1, fc2;
};

struct DecLayerW {
  const float *ln1g, *ln1b, *qkvb, *ob, *ln2g, *ln2b, *cqb, *cob, *ln3g, *ln3b, *fc1b, *fc2b;
  const __half *qkvw, *ow, *cqw, *cow, *fc1w, *fc2w;
};

// key of a captured step of the batched decoder pass
struct GraphKey {
  int n_utt, beam, prompt_len, max_new, max_hyp, u0, b_total, per_utt_max_new;
  int ts, ts_max_init;  // timestamp mode: the step graph bakes SearchArgs in, so a mode never reuses another's graph
  float lp;
  float rep_penalty;    // history processors (baked in too)
  int no_repeat_ngram;
  int mixed;            // per-utterance beam / max_hyp / length penalty in device arrays (beam = the largest; max_hyp, lp 0)
  int sample, topk;     // sampling (the seeds live in a device array: one graph serves every seed)
  float temperature;
  bool operator<(const GraphKey& o) const {
    return memcmp(this, &o, sizeof(GraphKey)) < 0;
  }
};

}  // namespace

}  // namespace wisb

using namespace wisb;

struct wisb_handle {
  int device = 0;
  int num_sms = 132;
  std::mutex mu;
  cudaStream_t stream = nullptr;
  Dims dims{};
  // weights
  uint8_t* blob = nullptr;
  bool own_blob = false;
  size_t blob_bytes = 0;
  std::map<std::string, TensorRef> tensors;
  std::vector<DecLayerW> dec_w;
  // options
  int use_graphs = 1, attn_v_mn = 1, attn_ref = 0;
  // front end
  DevBuf<float> lm_tables;
  DevBuf<unsigned> lm_max;
  DevBuf<uint8_t> pcm_dev;
  DevBuf<long long> pcm_off;
  DevBuf<int> pcm_n;
  DevBuf<float> mel;  // [B,n_mels,3000]
  int mel_B = 0;      // utterances currently held in `mel`
  // encoder output of enc_in_B windows from wisb_load_encoder_output, fp16 [enc_in_B, 1500, d].  While enc_in_B > 0 it,
  // not the features wisb_logmel kept, is what a call with mel == NULL decodes.
  DevBuf<__half> enc_in;
  int enc_in_B = 0;
  // encoder workspaces (capacity enc_cap utterances)
  int enc_cap = 0;
  DevBuf<__half> h1, xn, qkv, vt, ctx, hbuf, enc_out, ckv;
  DevBuf<float> x;
  GemmPlan plan_conv2, plan_ckv;
  CUtensorMap ckv_map;
  CUtensorMap ckv_map_plain;  // the same buffer without swizzle: reads the chunk-swizzled layout (wide prefill passes)
  std::vector<EncLayerPlans> enc_plans;
  AttnPlan attn_plan;
  int plans_B = 0, plans_vmn = -1, plans_pdl = -1;
  // decoder workspaces
  DevBuf<float> dx, dq, dctx, dh, logits;
  DevBuf<__half> dctx16, dh16, dxn16, dq16;
  DevBuf<float> dxstat;  // warp-MMA pass: fp16 exchange images of the attention output and the MLP hidden rows
  DevBuf<__half> kcache, vcache;  // [L][16][448][d]
  DevBuf<uint8_t> mask_base, mask_cur;
  std::vector<int> mask_extra;
  DevBuf<float> row_lse, cum, cand_score, best_score, lang_probs, part_max, part_sum;
  DevBuf<unsigned long long> part;
  DevBuf<int> cand_idx, tokens, seq0, seq1, ind0, ind1, flip, done, n_hyp, best_len, best_tokens, prompt_dev, lang_ids;
  DevBuf<DecState> st;
  DevBuf<int> row_pos, row_slot, max_new_u;
  DevBuf<int> prompt_fed;  // one word: SearchArgs::prompt_fed
  DevBuf<int> beam_u, max_hyp_u;  // per-utterance search options of a call that mixes them (SearchArgs::beam_u)
  DevBuf<float> lp_u;
  DevBuf<unsigned long long> seed_u;  // per-utterance seeds of a sampling call (SearchArgs::seed_u)
  int search_rows = 0;  // rows the search / state buffers above are sized for
  int search_gen = 0, bd_search_gen = -1;  // reallocation count of those buffers / the one the batched-pass plans were built for
  // batched decoder pass (more than DEC_MAX_ROWS rows): workspaces for bd_rows (multiple of 128) rows, bd_tcap positions
  int batch_rows = 320, batch_pdl = 1, decoder_batch = 1, cross_tc = 1, debug_chunk = 1;  // options: row capacity of one shared pass; programmatic dependent launch
  int bd_rows = 0, bd_tcap = 0, bd_launches_step = 0;
  DevBuf<float> bx, bq, bpart, blogits;
  DevBuf<__half> bxn, bctx, bh, bkc, bvc;
  std::vector<BatchLayer> bd_layers;
  GemmPlan bd_vocab;
  // wide prefill passes (more than 8 prompt positions per utterance in one pass, options "wide_prefill" / "prefill_rows"):
  // activation rows, row tables and GEMM plans of their own, so the decode step's workspaces and plans stay as they are.
  // pf_layers write K/V to pf_kc / pf_vc (layer stride pf_layer_cache, pf_tcap positions per slot); pf_rows is their
  // row capacity (multiple of 128).
  int wide_prefill = 1, prefill_rows = 1024;
  int pf_rows = 0, pf_tcap = 0;
  size_t pf_layer_cache = 0;
  const __half* pf_kc = nullptr;
  DevBuf<float> px, pq, ppart;
  DevBuf<__half> pxn, pctx, ph;
  DevBuf<int> ptok, ppos, pslot;
  std::vector<BatchLayer> pf_layers;
  // no-speech probability (option "no_speech_prob"): ns_prob [B] the call's values on the device, ns_host / ns_B the
  // last wisb_generate's on the host (ns_B 0: none).  A group's reductions each read their own row table, ns_used of
  // them staged so far in ns_pin / ns_rows.  Wide prefill: window u's final-LayerNorm row gathered into row u of ns_x
  // (ns_cap rows, a multiple of 128), ns_vocab its vocabulary GEMM into ns_logits.
  int no_speech = 0;
  DevBuf<float> ns_prob, ns_logits;
  DevBuf<int> ns_rows;
  PinBuf<int> ns_pin;
  int ns_used = 0;
  DevBuf<__half> ns_x;
  GemmPlan ns_vocab;
  int ns_cap = 0;
  std::vector<float> ns_host;
  int ns_B = 0;
  DevBuf<MegaLayer> mega_layers;
  DevBuf<__half> mega_img;  // warp-MMA pass: decoder weights as per-CTA shared-memory images (mega_mma_image)
  int enc_pdl = 1;  // encoder: programmatic dependent launch along the whole kernel chain (227 launches per window)
  int mega_mma = 1;  // 1: the warp-MMA persistent pass, 0: the SIMT persistent pass (option "mega_mma")
  DevBuf<unsigned> mega_flags;
  // optional reuse of the encoder output + cross K/V between consecutive calls on identical host features
  // (detect_language -> generate -> translate on one window, main.py:633-644, 514-547): option "encoder_cache"
  int encoder_cache = 0;
  std::vector<float> mel_cache;
  int mel_cache_B = 0;
  bool enc_valid = false;
  int ckv_is_sw = 0;  // layout of the cross K/V in HBM (1: chunk-swizzled, see ckv_layout)
  DevBuf<float> cross_part;
  DevBuf<unsigned> cross_flags;
  DevBuf<float> ln_fold;       // per LN-GEMV: s2[N] and folded bias[N] (qkv, cq, fc1 of every decoder layer, vocab)
  DevBuf<__half> fc2_chunked;  // decoder fc2 weights in chunk-major layout for the persistent pass kernel
  // wisb_align: alignment heads ordered by layer (al_items = their blob-order index, al_layer_off[l] = first of layer l),
  // the head of each, and the per-call workspaces
  std::vector<int> al_layer_off;
  int al_A = 0;
  DevBuf<int> al_items, al_head, al_ntext, al_nframes, al_text, al_path, al_len;
  DevBuf<float> al_cap, al_mat, al_probs;
  cudaEvent_t ev_flag[2] = {nullptr, nullptr};  // decode loop: `all_done` copies of the last two steps
  PinBuf<MegaLayer> mega_layers_host;
  PinBuf<int> pin_i;
  PinBuf<float> pin_f;
  PinBuf<uint8_t> pin_b;
  std::map<GraphKey, cudaGraphExec_t> graphs;
  // timing
  cudaEvent_t ev[8] = {};
  float timing[16] = {};
  int launches = 0;
  // optional per-kernel-family profile of the encoder (option "profile"): event pairs on the launching stream
  int profile = 0;
  std::vector<cudaEvent_t> prof_ev;
  std::vector<int> prof_cat;  // category of pair i: 0 gemm, 1 attention, 2 layernorm, 3 conv1
  size_t prof_used = 0;
  void prof_begin(int cat) {
    if (!profile) return;
    if (prof_used + 2 > prof_ev.size()) {
      cudaEvent_t a, b;
      WISB_CUDA(cudaEventCreate(&a));
      WISB_CUDA(cudaEventCreate(&b));
      prof_ev.push_back(a);
      prof_ev.push_back(b);
    }
    prof_cat.push_back(cat);
    WISB_CUDA(cudaEventRecord(prof_ev[prof_used], stream));
  }
  void prof_end() {
    if (!profile) return;
    WISB_CUDA(cudaEventRecord(prof_ev[prof_used + 1], stream));
    prof_used += 2;
  }
  void prof_collect() {  // call after a stream synchronize
    for (int i = 8; i < 16; ++i) timing[i] = 0.f;
    if (!profile) return;
    for (size_t i = 0; i + 1 < prof_used; i += 2) {
      float ms = 0.f;
      WISB_CUDA(cudaEventElapsedTime(&ms, prof_ev[i], prof_ev[i + 1]));
      const int cat = prof_cat[i / 2];
      timing[8 + cat] += ms;
      if (cat == 0) timing[12] += 1.f;
    }
    prof_used = 0;
    prof_cat.clear();
  }

  const TensorRef& T(const std::string& name) const {
    auto it = tensors.find(name);
    if (it == tensors.end()) throw Error(1, "weight blob is missing tensor '" + name + "'");
    return it->second;
  }
  const __half* H(const std::string& n) const { return reinterpret_cast<const __half*>(T(n).ptr); }
  const float* F(const std::string& n) const { return reinterpret_cast<const float*>(T(n).ptr); }
};

namespace {

constexpr int T_MAX = 448;

void parse_blob(wisb_handle* h, const std::vector<uint8_t>& head) {
  WISB_REQUIRE(head.size() >= 256 && memcmp(head.data(), "WISB200\0", 8) == 0, "not a WISB200 weight blob");
  uint32_t version, n_tensors;
  memcpy(&version, head.data() + 8, 4);
  memcpy(&n_tensors, head.data() + 12, 4);
  WISB_REQUIRE(version == 1, "unsupported weight blob version");
  memcpy(&h->dims, head.data() + 16, sizeof(Dims));
  WISB_REQUIRE(head.size() >= 256 + 96ull * n_tensors, "truncated weight blob table");
  for (uint32_t i = 0; i < n_tensors; ++i) {
    const uint8_t* e = head.data() + 256 + 96ull * i;
    char name[49] = {0};
    memcpy(name, e, 48);
    TensorRef t;
    uint32_t dt, nd;
    memcpy(&dt, e + 48, 4);
    memcpy(&nd, e + 52, 4);
    t.dtype = static_cast<int>(dt);
    t.ndim = static_cast<int>(nd);
    for (int k = 0; k < 4; ++k) {
      int64_t s;
      memcpy(&s, e + 56 + 8 * k, 8);
      t.shape[k] = s;
    }
    uint64_t off;
    memcpy(&off, e + 88, 8);
    WISB_REQUIRE(t.dtype >= 0 && t.dtype <= 2 && t.ndim >= 0 && t.ndim <= 4, "bad tensor dtype / rank in the weight blob");
    long long n_el = 1;
    for (int k = 0; k < 4; ++k) {
      WISB_REQUIRE(t.shape[k] >= 0 && t.shape[k] <= (1ll << 40), "bad tensor shape in the weight blob");
      n_el *= (k < t.ndim ? t.shape[k] : 1);
      WISB_REQUIRE(n_el <= (1ll << 40), "bad tensor shape in the weight blob");
    }
    const unsigned long long bytes = static_cast<unsigned long long>(n_el) * (t.dtype == 0 ? 2 : 4);
    WISB_REQUIRE(off <= h->blob_bytes && bytes <= h->blob_bytes - off, std::string("tensor '") + name + "' reaches outside the weight blob");
    t.ptr = h->blob + off;
    h->tensors[name] = t;
  }
  const Dims& d = h->dims;
  WISB_REQUIRE(d.d_model % 128 == 0 && d.d_model == 64 * d.n_heads && d.d_model <= 1536,
               "engine requires head_dim 64 and d_model a multiple of 128 (<= 1536)");
  WISB_REQUIRE((d.n_mels == 80 || d.n_mels == 128) && d.n_audio_ctx == T_ENC,
               "engine runs 80- or 128-bin log-mel features x 1500 positions");
  WISB_REQUIRE(d.n_text_ctx <= T_MAX, "n_text_ctx > 448");
  WISB_REQUIRE(d.n_langs <= 128, "more than 128 languages");
  WISB_REQUIRE(d.n_vocab > 0 && d.n_vocab_pad >= d.n_vocab && d.n_vocab_pad % 128 == 0 && d.n_enc_layers > 0 && d.n_dec_layers > 0,
               "bad vocabulary / layer counts in the weight blob");
  // every tensor the kernels index must have exactly the shape the dimensions imply (a truncated or mismatched blob
  // must fail here, not read out of bounds on the device)
  auto expect = [&](const std::string& name, int dtype, std::initializer_list<long long> shape) {
    auto it = h->tensors.find(name);
    WISB_REQUIRE(it != h->tensors.end(), "weight blob is missing tensor '" + name + "'");
    const TensorRef& t = it->second;
    bool ok = t.dtype == dtype && t.ndim == static_cast<int>(shape.size());
    int k = 0;
    for (long long v : shape) ok = ok && t.shape[k++] == v;
    WISB_REQUIRE(ok, "tensor '" + name + "' has the wrong dtype / shape for this model");
  };
  const long long dd = d.d_model;
  expect("enc.conv1.w", 0, {dd, 3ll * d.n_mels});
  expect("enc.conv2.w", 0, {dd, 3 * dd});
  expect("enc.pos", 1, {d.n_audio_ctx, dd});
  expect("dec.tok_emb", 0, {d.n_vocab_pad, dd});
  expect("dec.pos", 1, {d.n_text_ctx, dd});
  expect("dec.crosskv.w", 0, {2ll * d.n_dec_layers * dd, dd});
  expect("dec.crosskv.b", 1, {2ll * d.n_dec_layers * dd});
  for (int side = 0; side < 2; ++side) {
    const int nl = side == 0 ? d.n_enc_layers : d.n_dec_layers;
    for (int i = 0; i < nl; ++i) {
      const std::string p = std::string(side == 0 ? "enc." : "dec.") + std::to_string(i) + ".";
      expect(p + "qkv.w", 0, {3 * dd, dd});
      expect(p + "qkv.b", 1, {3 * dd});
      expect(p + "o.w", 0, {dd, dd});
      expect(p + "o.b", 1, {dd});
      expect(p + "fc1.w", 0, {4 * dd, dd});
      expect(p + "fc1.b", 1, {4 * dd});
      expect(p + "fc2.w", 0, {dd, 4 * dd});
      expect(p + "fc2.b", 1, {dd});
      expect(p + "ln1.g", 1, {dd});
      expect(p + "ln2.g", 1, {dd});
      if (side == 1) {
        expect(p + "cq.w", 0, {dd, dd});
        expect(p + "co.w", 0, {dd, dd});
        expect(p + "ln3.g", 1, {dd});
      }
    }
  }
  for (const char* nm : {"meta.suppress_ids", "meta.suppress_ids_begin"}) {
    auto it = h->tensors.find(nm);
    WISB_REQUIRE(it != h->tensors.end() && it->second.dtype == 2 && it->second.ndim <= 1, std::string("bad '") + nm + "' in the weight blob");
  }
}

void drop_graphs(wisb_handle* h) {
  for (auto& kv : h->graphs) cudaGraphExecDestroy(kv.second);
  h->graphs.clear();
}

// search / beam state for R rows (rows = utterances x beams of one shared decoder pass)
void ensure_search(wisb_handle* h, int rows) {
  if (rows <= h->search_rows) return;
  WISB_CUDA(cudaStreamSynchronize(h->stream));
  drop_graphs(h);  // captured graphs hold the old pointers
  const size_t R = static_cast<size_t>(rows);
  h->row_lse.ensure(R); h->cum.ensure(R);
  // (TOPK_CHUNKS + 1 chunks per row: timestamp mode adds one for the timestamp ids)
  h->part_max.ensure(R * (TOPK_CHUNKS + 1)); h->part_sum.ensure(R * (TOPK_CHUNKS + 1));
  h->part.ensure(R * (TOPK_CHUNKS + 1) * MAX_CAND);
  h->cand_score.ensure(R * MAX_CAND); h->cand_idx.ensure(R * MAX_CAND);
  h->tokens.ensure(R);
  h->seq0.ensure(R * T_MAX, true); h->seq1.ensure(R * T_MAX, true);
  h->ind0.ensure(R * T_MAX, true); h->ind1.ensure(R * T_MAX, true);
  h->done.ensure(R); h->n_hyp.ensure(R); h->best_score.ensure(R); h->best_len.ensure(R);
  h->best_tokens.ensure(R * T_MAX, true);
  h->prompt_dev.ensure(R * T_MAX);
  h->row_pos.ensure(R, true); h->row_slot.ensure(R, true); h->max_new_u.ensure(R, true);
  h->beam_u.ensure(R, true); h->max_hyp_u.ensure(R, true); h->lp_u.ensure(R, true);
  h->seed_u.ensure(R, true);
  h->lang_probs.ensure(R * 128);
  h->pin_i.ensure(4 + R * (T_MAX + 5));  // (upload_prompts: prompts and four per-utterance words)
  h->pin_f.ensure(R * 130);
  h->search_rows = rows;
  ++h->search_gen;  // whoever baked these pointers into plans must rebuild them
}

void finish_create(wisb_handle* h) {
  const Dims& d = h->dims;
  const bool has_model = h->blob != nullptr;
  cudaDeviceProp prop;
  WISB_CUDA(cudaGetDeviceProperties(&prop, h->device));
  WISB_REQUIRE(prop.major == 9 && prop.minor == 0, "libwisb200 is built for sm_90a (Hopper H100) only");
  h->num_sms = prop.multiProcessorCount;
  WISB_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  for (auto& e : h->ev) WISB_CUDA(cudaEventCreate(&e));
  h->lm_tables.ensure(logmel_table_floats());
  logmel_init_tables(h->lm_tables.p, d.n_mels, h->stream);
  if (!has_model) {  // front-end-only handle (wisb_create_frontend)
    WISB_CUDA(cudaStreamSynchronize(h->stream));
    return;
  }
  // per-layer decoder weight pointers
  h->dec_w.resize(d.n_dec_layers);
  for (int i = 0; i < d.n_dec_layers; ++i) {
    const std::string p = "dec." + std::to_string(i) + ".";
    DecLayerW& w = h->dec_w[i];
    w.ln1g = h->F(p + "ln1.g"); w.ln1b = h->F(p + "ln1.b");
    w.qkvw = h->H(p + "qkv.w"); w.qkvb = h->F(p + "qkv.b");
    w.ow = h->H(p + "o.w"); w.ob = h->F(p + "o.b");
    w.ln2g = h->F(p + "ln2.g"); w.ln2b = h->F(p + "ln2.b");
    w.cqw = h->H(p + "cq.w"); w.cqb = h->F(p + "cq.b");
    w.cow = h->H(p + "co.w"); w.cob = h->F(p + "co.b");
    w.ln3g = h->F(p + "ln3.g"); w.ln3b = h->F(p + "ln3.b");
    w.fc1w = h->H(p + "fc1.w"); w.fc1b = h->F(p + "fc1.b");
    w.fc2w = h->H(p + "fc2.w"); w.fc2b = h->F(p + "fc2.b");
  }
  // suppression mask: bit0 = always (suppress_ids), bit1 = at the first generated step (suppress_ids_begin)
  std::vector<uint8_t> mask(d.n_vocab, 0);
  auto fetch_ids = [&](const char* name) {
    const TensorRef& t = h->T(name);
    std::vector<int> ids(static_cast<size_t>(t.numel()));
    if (!ids.empty()) WISB_CUDA(cudaMemcpy(ids.data(), t.ptr, ids.size() * 4, cudaMemcpyDeviceToHost));
    return ids;
  };
  for (int id : fetch_ids("meta.suppress_ids"))
    if (id >= 0 && id < d.n_vocab) mask[id] |= 1;
  for (int id : fetch_ids("meta.suppress_ids_begin"))
    if (id >= 0 && id < d.n_vocab) mask[id] |= 2;
  {
    // alignment heads: meta.alignment_heads [A, 2] (layer, head), else every head of the upper half of the decoder
    std::vector<int> lh;
    auto it = h->tensors.find("meta.alignment_heads");
    if (it != h->tensors.end()) {
      const TensorRef& t = it->second;
      WISB_REQUIRE(t.dtype == 2 && t.ndim == 2 && t.shape[1] == 2 && t.shape[0] >= 1 && t.shape[0] <= 4096,
                   "bad 'meta.alignment_heads' in the weight blob");
      lh.resize(static_cast<size_t>(t.numel()));
      WISB_CUDA(cudaMemcpy(lh.data(), t.ptr, lh.size() * 4, cudaMemcpyDeviceToHost));
      for (size_t i = 0; i < lh.size(); i += 2)
        WISB_REQUIRE(lh[i] >= 0 && lh[i] < d.n_dec_layers && lh[i + 1] >= 0 && lh[i + 1] < d.n_heads,
                     "'meta.alignment_heads' names a head outside the decoder");
    } else {
      for (int l = d.n_dec_layers / 2; l < d.n_dec_layers; ++l)
        for (int hh = 0; hh < d.n_heads; ++hh) lh.insert(lh.end(), {l, hh});
    }
    const int A = static_cast<int>(lh.size() / 2);
    std::vector<int> items, heads(A);
    h->al_layer_off.assign(d.n_dec_layers + 1, 0);
    for (int l = 0; l < d.n_dec_layers; ++l) {
      h->al_layer_off[l] = static_cast<int>(items.size());
      for (int a = 0; a < A; ++a)
        if (lh[2 * a] == l) items.push_back(a);
    }
    h->al_layer_off[d.n_dec_layers] = A;
    for (int a = 0; a < A; ++a) heads[a] = lh[2 * a + 1];
    h->al_A = A;
    h->al_items.ensure(A);
    h->al_head.ensure(A);
    WISB_CUDA(cudaMemcpy(h->al_items.p, items.data(), A * 4, cudaMemcpyHostToDevice));
    WISB_CUDA(cudaMemcpy(h->al_head.p, heads.data(), A * 4, cudaMemcpyHostToDevice));
  }
  h->mask_base.ensure(d.n_vocab);
  h->mask_cur.ensure(d.n_vocab);
  WISB_CUDA(cudaMemcpy(h->mask_base.p, mask.data(), mask.size(), cudaMemcpyHostToDevice));
  WISB_CUDA(cudaMemcpy(h->mask_cur.p, mask.data(), mask.size(), cudaMemcpyHostToDevice));
  // decoder workspaces for DEC_MAX_ROWS rows (the persistent SIMT pass); the batched pass grows the search state later
  const size_t R = DEC_MAX_ROWS;
  h->dx.ensure(R * d.d_model, true);
  h->dq.ensure(R * d.d_model, true);
  h->dctx.ensure(R * d.d_model, true);
  h->dh.ensure(R * 4 * d.d_model, true);
  h->dctx16.ensure(R * d.d_model, true);
  h->dh16.ensure(R * 4 * d.d_model, true);
  h->dxn16.ensure(R * d.d_model, true);
  h->dq16.ensure(R * d.d_model, true);
  h->dxstat.ensure(static_cast<size_t>(h->num_sms) * R * 2, true);
  h->logits.ensure(R * d.n_vocab_pad, true);
  const size_t cache = static_cast<size_t>(d.n_dec_layers) * R * T_MAX * d.d_model;
  h->kcache.ensure(cache, true);
  h->vcache.ensure(cache, true);
  h->flip.ensure(1, true);
  h->st.ensure(1, true);
  h->prompt_fed.ensure(1, true);
  ensure_search(h, DEC_MAX_ROWS);
  h->mega_layers.ensure(d.n_dec_layers);
  h->mega_layers_host.ensure(d.n_dec_layers);
  h->mega_flags.ensure(mega_flags_words(), true);
  h->cross_flags.ensure(static_cast<size_t>(DEC_MAX_ROWS) * d.n_heads * 16 * 32, true);
  {
    // LayerNorm fold vectors for the persistent pass kernel (decoder_mega.cu consume_gemv)
    const size_t per_layer = 2ull * (3 * d.d_model + d.d_model + 4 * d.d_model);
    h->ln_fold.ensure(per_layer * d.n_dec_layers + 2ull * d.n_vocab_pad);
    for (int i = 0; i < d.n_dec_layers; ++i) {
      const DecLayerW& w = h->dec_w[i];
      float* base = h->ln_fold.p + per_layer * i;
      mega_ln_fold(w.qkvw, w.ln1g, w.ln1b, w.qkvb, base, base + 3 * d.d_model, 3 * d.d_model, d.d_model, h->stream);
      base += 6 * d.d_model;
      mega_ln_fold(w.cqw, w.ln2g, w.ln2b, w.cqb, base, base + d.d_model, d.d_model, d.d_model, h->stream);
      base += 2 * d.d_model;
      mega_ln_fold(w.fc1w, w.ln3g, w.ln3b, w.fc1b, base, base + 4 * d.d_model, 4 * d.d_model, d.d_model, h->stream);
    }
    float* vb = h->ln_fold.p + per_layer * d.n_dec_layers;
    mega_ln_fold(h->H("dec.tok_emb"), h->F("dec.ln.g"), h->F("dec.ln.b"), nullptr, vb, vb + d.n_vocab_pad, d.n_vocab, d.d_model, h->stream);
  }
  if (mega_k_chunks(4 * d.d_model) > 1) {
    const size_t per = static_cast<size_t>(4) * d.d_model * d.d_model;
    h->fc2_chunked.ensure(per * d.n_dec_layers);
    for (int i = 0; i < d.n_dec_layers; ++i)
      mega_chunk_major(h->dec_w[i].fc2w, h->fc2_chunked.p + per * i, d.d_model, 4 * d.d_model, h->stream);
  }
  h->cross_part.ensure(static_cast<size_t>(DEC_MAX_ROWS) * d.n_heads * 16 * MAX_BEAM * 68, true);
  if (4 * d.d_model <= 5120 && d.d_model % 64 == 0) {
    // warp-MMA pass: a second copy of the decoder weights laid out as the shared-memory image each CTA streams
    // (decoder_mega.cu mma_image_kernel); per layer qkv | o | cq | co | fc1 | fc2, then the vocabulary projection
    const size_t dd = d.d_model;
    const size_t per_layer = 14 * dd * dd;
    const size_t vocab_rows = static_cast<size_t>(d.n_vocab);
    h->mega_img.ensure(per_layer * d.n_dec_layers + vocab_rows * dd);
    for (int i = 0; i < d.n_dec_layers; ++i) {
      const DecLayerW& w = h->dec_w[i];
      __half* p = h->mega_img.p + per_layer * i;
      mega_mma_image(w.qkvw, p, 3 * d.d_model, d.d_model, h->num_sms, h->stream);
      mega_mma_image(w.ow, p + 3 * dd * dd, d.d_model, d.d_model, h->num_sms, h->stream);
      mega_mma_image(w.cqw, p + 4 * dd * dd, d.d_model, d.d_model, d.n_heads, h->stream);  // head-major: the cross phase projects its own queries
      mega_mma_image(w.cow, p + 5 * dd * dd, d.d_model, d.d_model, h->num_sms, h->stream);
      mega_mma_image(w.fc1w, p + 6 * dd * dd, 4 * d.d_model, d.d_model, h->num_sms, h->stream);
      mega_mma_image(w.fc2w, p + 10 * dd * dd, d.d_model, 4 * d.d_model, h->num_sms, h->stream);
    }
    mega_mma_image(h->H("dec.tok_emb"), h->mega_img.p + per_layer * d.n_dec_layers, d.n_vocab, d.d_model, h->num_sms, h->stream);
  } else {
    h->mega_mma = 0;
  }
  WISB_CUDA(cudaStreamSynchronize(h->stream));
}

// floats of the features of B windows: [B, n_mels, 3000]
size_t mel_floats(const wisb_handle* h, int B) { return static_cast<size_t>(B) * h->dims.n_mels * N_FRAMES; }

// feature buffer [B,n_mels,3000] (+ the per-utterance maxima of the log-mel kernel); growing it drops what it held
void ensure_mel(wisb_handle* h, int B) {
  h->lm_max.ensure(B);
  const size_t n = mel_floats(h, B);
  if (n <= h->mel.n) return;
  h->mel.ensure(n);
  h->mel_B = 0;
}

void ensure_encoder(wisb_handle* h, int B) {
  if (h->blob == nullptr) return;  // front-end-only handle
  const Dims& dm = h->dims;
  const int d = dm.d_model, H = dm.n_heads;
  const long long M = static_cast<long long>(B) * T_ENC_PAD;
  if (B > h->enc_cap) {
    h->plans_B = 0;
    drop_graphs(h);  // captured decoder graphs hold pointers into the buffers reallocated below
    h->h1.release();
    h->h1.ensure((static_cast<size_t>(B) * H1_ROWS + 8) * d, true);
    h->x.ensure(M * d, true);
    h->xn.ensure(M * d, true);
    h->qkv.ensure(M * 3 * d, true);
    h->vt.ensure(M * d, true);
    h->ctx.ensure(M * d, true);
    h->hbuf.ensure(M * 4 * d, true);
    h->enc_out.ensure(M * d, true);
    h->ckv.ensure(static_cast<size_t>(dm.n_dec_layers) * 2 * M * d, true);
    // the whole cross-K/V buffer as rows of one head's 64 values (for the wgmma cross-attention of the batched pass)
    make_tmap_f16_2d(&h->ckv_map, h->ckv.p, HEAD_DIM, static_cast<long long>(h->ckv.n / HEAD_DIM), HEAD_DIM, HEAD_DIM, 128);
    make_tmap_f16_2d_swizzle(&h->ckv_map_plain, h->ckv.p, HEAD_DIM, static_cast<long long>(h->ckv.n / HEAD_DIM), HEAD_DIM,
                             HEAD_DIM, 128, false);
    h->enc_cap = B;
  }
  // V stays in qkv (MN-major) unless the wgmma attention reads the transposed Vt: the SIMT attention (option
  // "attn_ref") reads V from qkv, which the Vt epilogue does not write
  const int vmn = h->attn_v_mn || h->attn_ref ? 1 : 0;
  if (h->plans_B == B && h->plans_vmn == vmn && h->plans_pdl == h->enc_pdl) return;
  const int Mi = static_cast<int>(M);
  {
    GemmEpi e;
    e.mode = EPI_CONV2;
    e.bias = h->F("enc.conv2.b");
    e.out = h->x.p;
    e.ldo = d;
    e.pos = h->F("enc.pos");
    gemm_plan(h->plan_conv2, h->h1.p, 2LL * d, h->H("enc.conv2.w"), Mi, d, 3 * d, e, h->num_sms, 0, 2 * d);
  }
  h->enc_plans.assign(dm.n_enc_layers, EncLayerPlans());
  for (int i = 0; i < dm.n_enc_layers; ++i) {
    const std::string p = "enc." + std::to_string(i) + ".";
    EncLayerPlans& pl = h->enc_plans[i];
    GemmEpi e;
    e.mode = vmn ? EPI_F16 : EPI_QKV_VT;
    e.bias = h->F(p + "qkv.b");
    e.out = h->qkv.p;
    e.ldo = 3 * d;
    e.aux = h->vt.p;
    e.d_model = d;
    e.n_heads = H;
    e.batch = B;
    gemm_plan(pl.qkv, h->xn.p, d, h->H(p + "qkv.w"), Mi, 3 * d, d, e, h->num_sms);
    GemmEpi eo;
    eo.mode = EPI_RESID_F32;
    eo.bias = h->F(p + "o.b");
    eo.out = h->x.p;
    eo.ldo = d;
    gemm_plan(pl.o, h->ctx.p, d, h->H(p + "o.w"), Mi, d, d, eo, h->num_sms);
    GemmEpi e1;
    e1.mode = EPI_F16_GELU;
    e1.bias = h->F(p + "fc1.b");
    e1.out = h->hbuf.p;
    e1.ldo = 4 * d;
    gemm_plan(pl.fc1, h->xn.p, d, h->H(p + "fc1.w"), Mi, 4 * d, d, e1, h->num_sms);
    GemmEpi e2;
    e2.mode = EPI_RESID_F32;
    e2.bias = h->F(p + "fc2.b");
    e2.out = h->x.p;
    e2.ldo = d;
    gemm_plan(pl.fc2, h->hbuf.p, 4LL * d, h->H(p + "fc2.w"), Mi, d, 4 * d, e2, h->num_sms);
  }
  {
    GemmEpi e;
    e.mode = EPI_CROSSKV;
    e.bias = h->F("dec.crosskv.b");
    e.out = h->ckv.p;
    e.d_model = d;
    e.n_heads = H;
    e.batch = B;
    gemm_plan(h->plan_ckv, h->enc_out.p, d, h->H("dec.crosskv.w"), Mi, dm.n_dec_layers * 2 * d, d, e, h->num_sms);
  }
  enc_attn_plan(h->attn_plan, h->qkv.p, h->vt.p, h->ctx.p, B, d, H, vmn != 0);
  h->attn_plan.pdl = h->enc_pdl != 0;
  h->plan_conv2.pdl = h->plan_ckv.pdl = h->enc_pdl;
  for (EncLayerPlans& pl : h->enc_plans) pl.qkv.pdl = pl.o.pdl = pl.fc1.pdl = pl.fc2.pdl = h->enc_pdl;
  h->plans_pdl = h->enc_pdl;
  h->plans_B = B;
  h->plans_vmn = vmn;
}

// decoder pass of a call on `rows` rows (utterances x beams): the persistent pass for <= 8 rows unless option
// "decoder_batch" = 2 forces the batched pass
bool use_persistent_pass(const wisb_handle* h, int rows) {
  return rows <= DEC_MAX_ROWS && h->decoder_batch != 2;
}

// cross-K/V layout the decoder pass reads: chunk-swizzled (1) for the persistent warp-MMA pass (ldmatrix without bank
// conflicts), linear (0) for the SIMT persistent pass, the batched pass and the alignment capture
int ckv_layout(const wisb_handle* h, bool persistent_pass) {
  return persistent_pass && h->mega_mma ? 1 : 0;
}

// Encoder stem on the plans ensure_encoder(h, B) bound: conv1 of windows [mel_first, mel_first + B) of h->mel into h1
// (rows 1..3000 of each window; row 0 and rows 3001.. stay zero from the allocation), then the conv2 GEMM into x.
void enc_stem_run(wisb_handle* h, int B, int mel_first) {
  cudaStream_t s = h->stream;
  h->prof_begin(3);
  conv1_gelu_run(h->mel.p + mel_floats(h, mel_first), h->H("enc.conv1.w"), h->F("enc.conv1.b"), h->h1.p, B,
                 h->dims.d_model, h->dims.n_mels, s);
  h->prof_end();
  h->prof_begin(0);
  gemm_run(h->plan_conv2, s);
  h->prof_end();
  h->launches += 2;
}

// The seven launches of encoder layer i on M = B * 1536 rows of x (plans of ensure_encoder(h, B)).  snap (debug entry
// only), if given, runs after launch k = 0..6 (LN1, QKV, attention, o-proj, LN2, fc1, fc2) and may read its output.
void enc_layer_run(wisb_handle* h, int i, int M, const std::function<void(int)>* snap) {
  const Dims& dm = h->dims;
  const int d = dm.d_model;
  cudaStream_t s = h->stream;
  const std::string p = "enc." + std::to_string(i) + ".";
  EncLayerPlans& pl = h->enc_plans[i];
  auto after = [&](int k) {
    if (snap) (*snap)(k);
  };
  h->prof_begin(2);
  layernorm_f32_to_f16_run(h->x.p, h->F(p + "ln1.g"), h->F(p + "ln1.b"), h->xn.p, M, d, s, h->enc_pdl != 0);
  h->prof_end();
  after(0);
  h->prof_begin(0);
  gemm_run(pl.qkv, s);
  h->prof_end();
  after(1);
  h->prof_begin(1);
  if (h->attn_ref)
    enc_attn_ref_run(h->qkv.p, h->ctx.p, M / T_ENC_PAD, d, dm.n_heads, s);
  else
    enc_attn_run(h->attn_plan, s);
  h->prof_end();
  after(2);
  h->prof_begin(0);
  gemm_run(pl.o, s);
  h->prof_end();
  after(3);
  h->prof_begin(2);
  layernorm_f32_to_f16_run(h->x.p, h->F(p + "ln2.g"), h->F(p + "ln2.b"), h->xn.p, M, d, s, h->enc_pdl != 0);
  h->prof_end();
  after(4);
  h->prof_begin(0);
  gemm_run(pl.fc1, s);
  h->prof_end();
  after(5);
  h->prof_begin(0);
  gemm_run(pl.fc2, s);
  h->prof_end();
  after(6);
  h->launches += 7;
}

// mel (device, [B,n_mels,3000]) -> enc_out fp16 [B*1536, d]
void run_encoder(wisb_handle* h, int B, int n_layers, int mel_first = 0) {
  const Dims& dm = h->dims;
  const int M = B * T_ENC_PAD;
  ensure_encoder(h, B);
  h->enc_valid = false;  // callers that want the result cached re-validate it after a full encode
  enc_stem_run(h, B, mel_first);
  const int nl = (n_layers < 0 || n_layers > dm.n_enc_layers) ? dm.n_enc_layers : n_layers;
  for (int i = 0; i < nl; ++i) enc_layer_run(h, i, M, nullptr);
  h->prof_begin(2);
  layernorm_f32_to_f16_run(h->x.p, h->F("enc.ln_post.g"), h->F("enc.ln_post.b"), h->enc_out.p, M, dm.d_model, h->stream,
                           h->enc_pdl != 0);
  h->prof_end();
  h->launches += 1;
}

// Places the features of this call in h->mel.  Returns true when the encoder output and cross K/V already in HBM belong
// to exactly these features (option "encoder_cache", host features of <= 2 windows compared byte for byte), in which
// case the caller skips the encoder.  Off by default: a benchmark that feeds the same utterance every step must not
// silently skip work.
bool upload_mel(wisb_handle* h, const float* mel, int B) {
  ensure_mel(h, B);
  if (mel == nullptr) {
    WISB_REQUIRE(h->mel_B == B, "mel == NULL but wisb_logmel(keep_on_device) did not leave features for this batch size");
    h->mel_cache_B = 0;
    return false;
  }
  const size_t n = mel_floats(h, B);
  if (h->encoder_cache && B <= 2) {
    if (h->enc_valid && h->mel_cache_B == B && memcmp(h->mel_cache.data(), mel, n * sizeof(float)) == 0) return true;
    h->mel_cache.assign(mel, mel + n);
    h->mel_cache_B = B;
  } else {
    h->mel_cache_B = 0;
  }
  h->enc_valid = false;
  WISB_CUDA(cudaMemcpyAsync(h->mel.p, mel, n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  h->mel_B = B;
  return false;
}

// True when a call with these arguments decodes the encoder output wisb_load_encoder_output loaded: mel == NULL after
// that call rather than after wisb_logmel(keep_on_device).  The call must then have the loaded batch size.
bool loaded_source(const wisb_handle* h, const float* mel, int B) {
  if (mel != nullptr || h->enc_in_B == 0) return false;
  WISB_REQUIRE(h->enc_in_B == B, "mel == NULL but wisb_load_encoder_output loaded an encoder output of another batch size");
  return true;
}

// `p` must be device memory on the handle's device (wisb_encode's out, wisb_load_encoder_output's enc)
void require_on_device(const wisb_handle* h, const void* p, const char* what) {
  cudaPointerAttributes a{};
  WISB_CUDA(cudaPointerGetAttributes(&a, p));
  WISB_REQUIRE(a.type == cudaMemoryTypeDevice && a.device == h->device,
               std::string(what) + " is not device memory on the handle's device");
}

// Encoder stage of a call on the B windows placed by upload_mel: leaves the encoder output and the cross K/V of windows
// [g0, g0 + n) in HBM, the cross K/V in layout `ckv_sw` (ckv_layout).  What is already there is reused only when
// upload_mel reported a hit (`cached`) and this group is the whole call (the cache holds a batch of B windows); cached
// cross K/V in the other layout is rewritten by the cross-K/V GEMM alone.  With `loaded` (loaded_source) the group's rows
// of the loaded encoder output take the encoder's place.  Records the stage events ev[2] (start), ev[3] (encoder done)
// and ev[4] (cross K/V done).
void encode_stage(wisb_handle* h, bool cached, bool loaded, int B, int g0, int n, int ckv_sw) {
  cudaStream_t s = h->stream;
  const bool reuse = cached && n == B;
  WISB_CUDA(cudaEventRecord(h->ev[2], s));
  if (loaded) {
    // rows [g0, g0 + n) into enc_out's padded layout; padding rows 1500..1535 are zero (the cross-attention masks keys
    // >= 1500, so they never reach a result).  These rows belong to no features: the encoder cache must not claim them.
    ensure_encoder(h, n);
    h->enc_valid = false;
    h->mel_cache_B = 0;
    const size_t row = static_cast<size_t>(h->dims.d_model) * sizeof(__half);
    WISB_CUDA(cudaMemcpy2DAsync(h->enc_out.p, T_ENC_PAD * row, h->enc_in.p + static_cast<size_t>(g0) * T_ENC * h->dims.d_model,
                                T_ENC * row, T_ENC * row, n, cudaMemcpyDeviceToDevice, s));
    WISB_CUDA(cudaMemset2DAsync(reinterpret_cast<char*>(h->enc_out.p) + T_ENC * row, T_ENC_PAD * row, 0,
                                (T_ENC_PAD - T_ENC) * row, n, s));
  } else if (!reuse) {
    run_encoder(h, n, -1, g0);
  }
  WISB_CUDA(cudaEventRecord(h->ev[3], s));
  if (!reuse || h->ckv_is_sw != ckv_sw) {
    ensure_encoder(h, n);
    h->prof_begin(0);
    h->plan_ckv.epi.kv_swizzle = ckv_sw;
    gemm_run(h->plan_ckv, s);
    h->prof_end();
    h->ckv_is_sw = ckv_sw;
    h->launches += 1;
  }
  if (!reuse) h->enc_valid = h->encoder_cache != 0 && h->mel_cache_B == B && n == B;
  WISB_CUDA(cudaEventRecord(h->ev[4], s));
}

// Stage timings of wisb_generate / wisb_align (slots as documented in wisb200.h).  ev[0] opens the call, ev[1] closes its
// host-to-device stage, and ev[2], ev[3], ... delimit the stages of one group of utterances (encode_stage records ev[2]
// to ev[4], the caller the rest).
void time_h2d(wisb_handle* h) {
  WISB_CUDA(cudaEventRecord(h->ev[1], h->stream));
  WISB_CUDA(cudaEventSynchronize(h->ev[1]));
  WISB_CUDA(cudaEventElapsedTime(&h->timing[1], h->ev[0], h->ev[1]));
}

// after the last stage of a group: adds the time from ev[2 + k] to ev[3 + k] to timing[slots[k]] and sets timing[5], the
// call's total so far (ev[0] to the group's last event)
void time_group(wisb_handle* h, std::initializer_list<int> slots) {
  const cudaEvent_t* e = h->ev + 2;
  WISB_CUDA(cudaEventSynchronize(e[slots.size()]));
  for (int slot : slots) {
    float t;
    WISB_CUDA(cudaEventElapsedTime(&t, e[0], e[1]));
    h->timing[slot] += t;
    ++e;
  }
  WISB_CUDA(cudaEventElapsedTime(&h->timing[5], h->ev[0], *e));
}

struct DecodeCfg {
  int u0, n_utt, B_total, beam, prompt_len, max_new, max_hyp;
  float lp;
  int per_utt_max_new = 0;  // h->max_new_u holds a per-utterance cap (<= max_new)
  int ts = 0;               // timestamp rules on (the prompt has no <|notimestamps|>)
  int ts_max_init = 0;      // max_initial_timestamp_index
  float rep_penalty = 1.f;  // repetition_penalty (1 = off)
  int no_repeat_ngram = 0;  // no_repeat_ngram_size (0 = off)
  // per-utterance search options (host arrays indexed like max_new_host, from u0): beam is then the largest of beam_host
  // over the slice, and max_hyp / lp are unused
  int mixed = 0;
  const int* beam_host = nullptr;
  const int* max_hyp_host = nullptr;
  const float* lp_host = nullptr;
  // sampling: beam is the number of hypotheses per utterance, seeds (host, indexed like max_new_host) -> h->seed_u
  int sample = 0, topk = 0;
  float temperature = 1.f;
  const uint64_t* seed_host = nullptr;
  // no-speech probability requested: sot[u] (host) = the position of the first <|startoftranscript|> in utterance u's
  // prompt, ns_out (device) [n_utt] its value; null: not requested
  const int* sot = nullptr;
  float* ns_out = nullptr;
};

SearchArgs make_search_args(wisb_handle* h, const DecodeCfg& c) {
  const Dims& dm = h->dims;
  SearchArgs a;
  a.logits = h->logits.p;
  a.ldl = dm.n_vocab_pad;
  a.n_vocab = dm.n_vocab;
  a.mask = h->mask_cur.p;
  a.n_utt = c.n_utt;
  a.beam = c.beam;
  a.n_cand = 2 * c.beam;
  a.max_new = c.max_new;
  a.max_hyp = c.max_hyp;
  a.eot = dm.eot;
  a.t_max = T_MAX;
  a.prompt_len = c.prompt_len;
  a.length_penalty = c.lp;
  a.row_lse = h->row_lse.p;
  a.part_max = h->part_max.p;
  a.part_sum = h->part_sum.p;
  a.cum = h->cum.p;
  a.part = h->part.p;
  a.cand_score = h->cand_score.p;
  a.cand_idx = h->cand_idx.p;
  a.tokens = h->tokens.p;
  a.seq[0] = h->seq0.p;
  a.seq[1] = h->seq1.p;
  a.indir[0] = h->ind0.p;
  a.indir[1] = h->ind1.p;
  a.flip = h->flip.p;
  a.done = h->done.p;
  a.n_hyp = h->n_hyp.p;
  a.best_score = h->best_score.p;
  a.best_len = h->best_len.p;
  a.best_tokens = h->best_tokens.p;
  a.st = h->st.p;
  a.row_pos = h->row_pos.p;
  a.row_slot = h->row_slot.p;
  a.prompt_fed = h->prompt_fed.p;
  a.max_new_u = c.per_utt_max_new ? h->max_new_u.p : nullptr;
  a.rep_penalty = c.rep_penalty;
  a.no_repeat_ngram = c.no_repeat_ngram;
  if (c.mixed) {
    a.beam_u = h->beam_u.p;
    a.max_hyp_u = h->max_hyp_u.p;
    a.lp_u = h->lp_u.p;
  }
  if (c.sample) {
    a.sample = 1;
    a.topk = c.topk;
    a.temperature = c.temperature;
    a.seed_u = h->seed_u.p;
  }
  if (c.ts) {
    a.ts = 1;
    a.no_ts = dm.no_timestamps;
    a.ts_begin = dm.no_timestamps + 1;
    a.ts_max_init = std::min(a.ts_begin + c.ts_max_init, dm.n_vocab - 1);
  }
  return a;
}

// points a layer descriptor (MegaLayer / BatchLayer) at the cross K and V of decoder layer `layer` for utterance u0 of a
// batch of B_total encoded windows (h->ckv: [layer][K | V][B_total][H][1536][64])
template <typename Layer>
void bind_cross_kv(const wisb_handle* h, Layer& l, int layer, int u0, int B_total) {
  const size_t head_block = static_cast<size_t>(h->dims.n_heads) * T_ENC_PAD * HEAD_DIM;
  l.ck = h->ckv.p + (static_cast<size_t>(layer * 2 + 0) * B_total + u0) * head_block;
  l.cv = h->ckv.p + (static_cast<size_t>(layer * 2 + 1) * B_total + u0) * head_block;
}

// descriptors of the persistent decoder pass for this batch slice (device array of per-layer pointers)
void upload_mega_layers(wisb_handle* h, const DecodeCfg& c) {
  const Dims& dm = h->dims;
  const int d = dm.d_model;
  const size_t layer_cache = static_cast<size_t>(DEC_MAX_ROWS) * T_MAX * d;
  for (int i = 0; i < dm.n_dec_layers; ++i) {
    const DecLayerW& w = h->dec_w[i];
    MegaLayer& m = h->mega_layers_host.p[i];
    m = MegaLayer();
    // (LayerNorm-fused GEMVs: `bias` is the folded bias, ln_s2 the fold vector, both precomputed at load)
    auto set = [&](MegaGemv& g, const __half* wt, const float* bias, const float* lg, const float* s2, const float* x,
                   float* out, long long ldo, int N, int K, int epi) {
      g.w = wt; g.bias = bias; g.ln_g = lg; g.ln_s2 = s2; g.x = x; g.out = out; g.ldo = ldo; g.N = N; g.K = K; g.epi = epi;
    };
    const size_t per_layer = 2ull * (3 * d + d + 4 * d);
    const float* fb = h->ln_fold.p + per_layer * i;
    set(m.qkv, w.qkvw, fb + 3 * d, w.ln1g, fb, h->dx.p, h->dq.p, d, 3 * d, d, GV_QKV);
    set(m.o, w.ow, w.ob, nullptr, nullptr, h->dctx.p, h->dx.p, d, d, d, GV_RESID);
    set(m.cq, w.cqw, fb + 7 * d, w.ln2g, fb + 6 * d, h->dx.p, h->dq.p, d, d, d, GV_STORE);
    set(m.co, w.cow, w.cob, nullptr, nullptr, h->dctx.p, h->dx.p, d, d, d, GV_RESID);
    set(m.fc1, w.fc1w, fb + 12 * d, w.ln3g, fb + 8 * d, h->dx.p, h->dh.p, 4 * d, 4 * d, d, GV_GELU);
    const __half* fc2w = (h->fc2_chunked.p && !h->mega_mma) ? h->fc2_chunked.p + static_cast<size_t>(4) * d * d * i : w.fc2w;
    set(m.fc2, fc2w, w.fc2b, nullptr, nullptr, h->dh.p, h->dx.p, d, d, 4 * d, GV_RESID);
    if (h->mega_mma) {
      m.o.x16 = h->dctx16.p;
      m.co.x16 = h->dctx16.p;
      m.fc1.out16 = h->dh16.p;
      m.fc2.x16 = h->dh16.p;
      m.qkv.x16 = m.cq.x16 = m.fc1.x16 = h->dxn16.p;
      m.cq.out16 = h->dq16.p;
      m.qkv.shape = 0;
      m.o.shape = m.cq.shape = m.co.shape = 1;
      m.fc1.shape = 2;
      m.fc2.shape = 3;
      m.o.next_g = w.ln2g;
      m.co.next_g = w.ln3g;
      m.fc2.next_g = i + 1 < dm.n_dec_layers ? h->dec_w[i + 1].ln1g : h->F("dec.ln.g");
      const size_t dd = d;
      const __half* img = h->mega_img.p + 14 * dd * dd * i;
      m.qkv.w = img;
      m.o.w = img + 3 * dd * dd;
      m.cq.w = img + 4 * dd * dd;
      m.co.w = img + 5 * dd * dd;
      m.fc1.w = img + 6 * dd * dd;
      m.fc2.w = img + 10 * dd * dd;
    }
    bind_cross_kv(h, m, i, c.u0, c.B_total);
    m.kcache = h->kcache.p + i * layer_cache;
    m.vcache = h->vcache.p + i * layer_cache;
  }
  WISB_CUDA(cudaMemcpyAsync(h->mega_layers.p, h->mega_layers_host.p, sizeof(MegaLayer) * dm.n_dec_layers,
                            cudaMemcpyHostToDevice, h->stream));
}

// one decoder forward for R <= 8 rows at position st->pos: ONE launch of the persistent pass.  pf_len > 0: prompt
// positions [0, pf_len) of every utterance instead (with_logits: logits of every one of those rows)
void enqueue_decoder_forward(wisb_handle* h, const DecodeCfg& c, bool with_logits, int pf_len = 0) {
  const Dims& dm = h->dims;
  MegaArgs a;
  a.layers = h->mega_layers.p;
  a.n_layers = dm.n_dec_layers;
  a.vocab.w = h->H("dec.tok_emb");
  a.vocab.ln_g = h->F("dec.ln.g");
  {
    const size_t per_layer = 2ull * 8 * dm.d_model;
    const float* vb = h->ln_fold.p + per_layer * dm.n_dec_layers;
    a.vocab.ln_s2 = vb;
    a.vocab.bias = vb + dm.n_vocab_pad;
  }
  a.vocab.x = h->dx.p;
  a.vocab.out = h->logits.p;
  a.vocab.ldo = dm.n_vocab_pad;
  a.vocab.N = dm.n_vocab;
  a.vocab.K = dm.d_model;
  a.vocab.epi = GV_STORE;
  if (h->mega_mma) {
    a.vocab.w = h->mega_img.p + static_cast<size_t>(14) * dm.d_model * dm.d_model * dm.n_dec_layers;
    a.tc = 1;
    a.ctx16 = h->dctx16.p;
    a.xn16 = h->dxn16.p;
    a.q16 = h->dq16.p;
    a.xstat = h->dxstat.p;
    a.vocab.x16 = h->dxn16.p;
    a.vocab.shape = 4;
  }
  a.with_logits = with_logits ? 1 : 0;
  a.R = c.n_utt * c.beam;
  a.d = dm.d_model;
  a.H = dm.n_heads;
  a.n_utt = c.n_utt;
  a.beam = c.beam;
  a.t_max = T_MAX;
  a.tokens = h->tokens.p;
  if (pf_len > 0) {  // the prompt positions of every utterance in ONE pass (rows = utterances x positions)
    a.pf_len = pf_len;
    a.pf_tok_stride = c.prompt_len;
    a.pf_slot_stride = c.beam;
    a.R = c.n_utt * a.pf_len;
    a.beam = a.pf_len;
    a.tokens = h->prompt_dev.p;
  }
  a.tok_emb = h->H("dec.tok_emb");
  a.pos_emb = h->F("dec.pos");
  a.x = h->dx.p;
  a.q = h->dq.p;
  a.ctx = h->dctx.p;
  a.indir0 = h->ind0.p;
  a.indir1 = h->ind1.p;
  a.flip = h->flip.p;
  a.st = h->st.p;
  a.cross_part = h->cross_part.p;
  a.cross_flags = h->cross_flags.p;
  a.epoch_base = h->mega_flags.p;
  dec_pass_run(a, h->num_sms, h->stream);
}

void enqueue_prefill(wisb_handle* h, const DecodeCfg& c, bool with_logits = false) {
  enqueue_decoder_forward(h, c, with_logits);
  prefill_advance_run(h->tokens.p, h->prompt_dev.p, c.prompt_len, c.n_utt * c.beam, c.beam, h->st.p, h->stream);
}
void enqueue_step(wisb_handle* h, const DecodeCfg& c) {
  enqueue_decoder_forward(h, c, true);
  search_step_run(make_search_args(h, c), h->stream);
}

void set_extra_suppress(wisb_handle* h, const int32_t* extra, int n_extra) {
  std::vector<int> want(extra ? extra : nullptr, extra ? extra + n_extra : nullptr);
  if (want == h->mask_extra) return;
  const Dims& dm = h->dims;
  for (int id : want) WISB_REQUIRE(id >= 0 && id < dm.n_vocab, "suppress token id outside the vocabulary");
  h->mask_extra.assign(1, -1);  // not a valid set: if anything below fails, the next call rebuilds the mask
  WISB_CUDA(cudaMemcpyAsync(h->mask_cur.p, h->mask_base.p, dm.n_vocab, cudaMemcpyDeviceToDevice, h->stream));
  if (!want.empty()) {
    std::vector<uint8_t> m(dm.n_vocab);
    WISB_CUDA(cudaMemcpyAsync(m.data(), h->mask_base.p, dm.n_vocab, cudaMemcpyDeviceToHost, h->stream));
    WISB_CUDA(cudaStreamSynchronize(h->stream));
    for (int id : want) m[id] |= 1;
    WISB_CUDA(cudaMemcpyAsync(h->mask_cur.p, m.data(), dm.n_vocab, cudaMemcpyHostToDevice, h->stream));
    WISB_CUDA(cudaStreamSynchronize(h->stream));
  }
  h->mask_extra = want;
}

// prompts [n_utt][prompt_len] of utterances [u0, u0 + n_utt) -> h->prompt_dev, when c.per_utt_max_new their caps on
// new tokens (max_new_host[u0 + u]) -> h->max_new_u, when c.mixed their search options -> h->beam_u / max_hyp_u /
// lp_u, and when c.sample their seeds -> h->seed_u.  All are staged through the pinned buffer, whose first 4 words hold
// the step loop's flags: the host may rewrite it only after the stream sync that ends the previous group, because these
// asynchronous copies read from it.
void upload_prompts(wisb_handle* h, const int32_t* prompts, const int* max_new_host, const DecodeCfg& c) {
  const size_t n = static_cast<size_t>(c.n_utt) * c.prompt_len;
  int* pin = h->pin_i.p + 4;
  memcpy(pin, prompts + static_cast<size_t>(c.u0) * c.prompt_len, sizeof(int) * n);
  WISB_CUDA(cudaMemcpyAsync(h->prompt_dev.p, pin, sizeof(int) * n, cudaMemcpyHostToDevice, h->stream));
  if (c.per_utt_max_new) {
    memcpy(pin + n, max_new_host + c.u0, sizeof(int) * c.n_utt);
    WISB_CUDA(cudaMemcpyAsync(h->max_new_u.p, pin + n, sizeof(int) * c.n_utt, cudaMemcpyHostToDevice, h->stream));
  }
  if (c.mixed) {
    int* pm = pin + n + c.n_utt;
    memcpy(pm, c.beam_host + c.u0, sizeof(int) * c.n_utt);
    memcpy(pm + c.n_utt, c.max_hyp_host + c.u0, sizeof(int) * c.n_utt);
    memcpy(pm + 2 * c.n_utt, c.lp_host + c.u0, sizeof(float) * c.n_utt);
    WISB_CUDA(cudaMemcpyAsync(h->beam_u.p, pm, sizeof(int) * c.n_utt, cudaMemcpyHostToDevice, h->stream));
    WISB_CUDA(cudaMemcpyAsync(h->max_hyp_u.p, pm + c.n_utt, sizeof(int) * c.n_utt, cudaMemcpyHostToDevice, h->stream));
    WISB_CUDA(cudaMemcpyAsync(h->lp_u.p, pm + 2 * c.n_utt, sizeof(float) * c.n_utt, cudaMemcpyHostToDevice, h->stream));
  }
  if (c.sample) {  // (never together with c.mixed: the same staging words)
    int* ps = pin + n + c.n_utt;
    memcpy(ps, c.seed_host + c.u0, sizeof(uint64_t) * c.n_utt);
    WISB_CUDA(cudaMemcpyAsync(h->seed_u.p, ps, sizeof(uint64_t) * c.n_utt, cudaMemcpyHostToDevice, h->stream));
  }
}

// best hypothesis of every utterance of the pass (search state) -> the caller's host arrays at utterance u0.  An
// utterance capped at 0 new tokens (c.max_new or its max_new_host entry) returns no tokens and score 0.
void read_results(wisb_handle* h, const DecodeCfg& c, const int* max_new_host, int32_t* out_ids, int out_stride,
                  int32_t* out_len, float* out_score) {
  cudaStream_t s = h->stream;
  if (c.sample) {
    // sampling: the hypothesis of every row; utterance u's n = c.beam go to entries (u0 + u) * n + [0, n), sorted by
    // score, descending, ties to the lower hypothesis index
    const int n = c.beam, R = c.n_utt * n;
    int* lens = h->pin_i.p + 4;
    int* toks = lens + R;
    const int mn = c.max_new > 0 ? c.max_new : 1;
    WISB_CUDA(cudaMemcpyAsync(lens, h->best_len.p, sizeof(int) * R, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(toks, h->best_tokens.p, sizeof(int) * R * mn, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(h->pin_f.p, h->best_score.p, sizeof(float) * R, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
    std::vector<int> order(n);
    for (int u = 0; u < c.n_utt; ++u) {
      const int cap = c.per_utt_max_new ? max_new_host[c.u0 + u] : c.max_new;
      const float* sc = h->pin_f.p + u * n;
      for (int k = 0; k < n; ++k) order[k] = k;
      if (cap > 0) std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return sc[x] > sc[y]; });
      for (int i = 0; i < n; ++i) {
        const int k = order[i], r = u * n + k;
        const size_t o = static_cast<size_t>(c.u0 + u) * n + i;
        const int len = cap > 0 ? lens[r] : 0;
        out_len[o] = len;
        for (int t = 0; t < len && t < out_stride; ++t) out_ids[o * out_stride + t] = toks[static_cast<size_t>(r) * mn + t];
        if (out_score) out_score[o] = cap > 0 ? sc[k] : 0.f;
      }
    }
    return;
  }
  int* lens = h->pin_i.p + 4;
  int* toks = lens + c.n_utt;
  const int mn = c.max_new > 0 ? c.max_new : 1;
  WISB_CUDA(cudaMemcpyAsync(lens, h->best_len.p, sizeof(int) * c.n_utt, cudaMemcpyDeviceToHost, s));
  WISB_CUDA(cudaMemcpyAsync(toks, h->best_tokens.p, sizeof(int) * c.n_utt * mn, cudaMemcpyDeviceToHost, s));
  WISB_CUDA(cudaMemcpyAsync(h->pin_f.p, h->best_score.p, sizeof(float) * c.n_utt, cudaMemcpyDeviceToHost, s));
  WISB_CUDA(cudaStreamSynchronize(s));
  for (int u = 0; u < c.n_utt; ++u) {
    const int cap = c.per_utt_max_new ? max_new_host[c.u0 + u] : c.max_new;
    const int len = cap > 0 ? lens[u] : 0;
    out_len[c.u0 + u] = len;
    for (int t = 0; t < len && t < out_stride; ++t) out_ids[static_cast<size_t>(c.u0 + u) * out_stride + t] = toks[u * mn + t];
    if (out_score) out_score[c.u0 + u] = cap > 0 ? h->pin_f.p[u] : 0.f;
  }
}

// setup of the persistent pass for this batch slice: prompts (and caps), search state (`fed` prompt positions forwarded
// by one prefill pass, search_init_run), layer descriptors
void persistent_setup(wisb_handle* h, const DecodeCfg& c, const int32_t* prompts, const int* max_new_host, int fed = 0) {
  upload_prompts(h, prompts, max_new_host, c);
  search_init_run(make_search_args(h, c), h->prompt_dev.p, h->stream, fed);
  upload_mega_layers(h, c);
}

// Generated-token loop of both decoder passes: enqueue(gs) issues step gs and returns its kernel launches; the loop ends at
// the first step whose `all_done` word reads 1.  With look_ahead (the persistent pass) step gs + 1 is enqueued BEFORE the
// host waits for step gs's word (the kernels of a step that turns out to be superfluous leave at once on the device flag),
// so neither the launch latency of the cooperative kernel nor the host's wake-up sits between two steps.  The batched
// pass polls after every step instead: its GEMMs do not exit early.  Returns the steps that did work.
int step_loop(wisb_handle* h, int max_new, bool look_ahead, const std::function<int(int gs)>& enqueue) {
  cudaStream_t s = h->stream;
  volatile int* flag = h->pin_i.p;
  flag[0] = flag[1] = 0;
  if (look_ahead && h->ev_flag[0] == nullptr) {
    WISB_CUDA(cudaEventCreateWithFlags(&h->ev_flag[0], cudaEventDisableTiming));
    WISB_CUDA(cudaEventCreateWithFlags(&h->ev_flag[1], cudaEventDisableTiming));
  }
  int steps = 0;
  for (int gs = 0; gs < max_new; ++gs) {
    h->launches += enqueue(gs);
    ++steps;
    WISB_CUDA(cudaMemcpyAsync(const_cast<int*>(flag) + (gs & 1), &h->st.p->all_done, sizeof(int), cudaMemcpyDeviceToHost, s));
    if (!look_ahead) {
      WISB_CUDA(cudaStreamSynchronize(s));
      if (flag[gs & 1]) break;
      continue;
    }
    WISB_CUDA(cudaEventRecord(h->ev_flag[gs & 1], s));
    if (gs >= 1) {
      WISB_CUDA(cudaEventSynchronize(h->ev_flag[(gs - 1) & 1]));
      if (flag[(gs - 1) & 1]) {
        --steps;  // the step just enqueued does nothing
        break;
      }
    }
  }
  return steps;
}

int wide_prefill_ns(wisb_handle* h, const DecodeCfg& c, int chunk, __half* kc, __half* vc, size_t layer_cache, int t_cap);

// ------------------------------------------------------------------------------------------------- no-speech probability
// openai/whisper's no_speech_prob: softmax of the raw logits at each window's first <|startoftranscript|> position s_u,
// at <|nospeech|>.  Whichever pass first forwards s_u also yields that row's logits (or, for a wide prefill pass, its
// final-LayerNorm row); the passes themselves are the ones the call runs without the request.

// whether some utterance's s_u lies in [lo, hi)
bool ns_in(const DecodeCfg& c, int lo, int hi) {
  if (c.sot == nullptr) return false;
  for (int u = 0; u < c.n_utt; ++u)
    if (c.sot[u] >= lo && c.sot[u] < hi) return true;
  return false;
}

// row tables of one group: at most one reduction per pass that forwards some s_u, the wide gather's and the first step's
void ns_begin(wisb_handle* h, const DecodeCfg& c) {
  h->ns_used = 0;
  if (c.sot == nullptr) return;
  const size_t n = static_cast<size_t>(c.n_utt) * (std::min(c.n_utt, c.prompt_len) + 2);
  h->ns_pin.ensure(n);  // (the previous group's copies from it ended with that group's synchronise)
  h->ns_rows.ensure(n);
}

// row(u) for every utterance, in a row table of its own (the group's copies are in flight together) -> its device
// address, or null when no utterance has a row here
const int* ns_table(wisb_handle* h, const DecodeCfg& c, const std::function<int(int u)>& row) {
  if (c.sot == nullptr) return nullptr;
  const size_t off = static_cast<size_t>(h->ns_used) * c.n_utt;
  WISB_REQUIRE(off + c.n_utt <= h->ns_rows.n, "no-speech: more reductions than the group's row tables hold");
  int* t = h->ns_pin.p + off;
  bool any = false;
  for (int u = 0; u < c.n_utt; ++u) any |= (t[u] = row(u)) >= 0;
  if (!any) return nullptr;
  ++h->ns_used;
  WISB_CUDA(cudaMemcpyAsync(h->ns_rows.p + off, t, sizeof(int) * c.n_utt, cudaMemcpyHostToDevice, h->stream));
  return h->ns_rows.p + off;
}

// c.ns_out[u] from row row(u) of logits (row(u) < 0: not in this buffer)
void ns_reduce(wisb_handle* h, const DecodeCfg& c, const float* logits, const std::function<int(int u)>& row) {
  const int* t = ns_table(h, c, row);
  if (t == nullptr) return;
  no_speech_run(logits, h->dims.n_vocab_pad, t, c.n_utt, h->dims.n_vocab, h->dims.no_speech, c.ns_out, h->stream);
  ++h->launches;
}

// the rows of the first decoding step's pass (utterance u's first beam) for every utterance whose prompt ends at s_u
void ns_reduce_first_step(wisb_handle* h, const DecodeCfg& c, const float* logits) {
  const int P = c.prompt_len;
  ns_reduce(h, c, logits, [&](int u) { return c.sot[u] == P - 1 ? u * c.beam : -1; });
}

// decode utterances [u0, u0 + n_utt) of the encoded batch with the persistent pass (<= 8 rows); writes results to the
// host arrays
int decode_pass(wisb_handle* h, const DecodeCfg& c, const int32_t* prompts, const int* max_new_host, int32_t* out_ids,
                int out_stride, int32_t* out_len, float* out_score) {
  int steps = 0;
  const int P = c.prompt_len;
  // every prompt position of every utterance fits one pass of the 8-row kernel: that pass also yields the logits of the
  // first step, which then runs no pass of its own
  const bool fused = c.n_utt * P <= DEC_MAX_ROWS && P <= MAX_BEAM;
  // else the prompt prefix (all but the last token) in one pass when it fits
  const bool one_pass_prefill = !fused && P > 1 && c.n_utt * (P - 1) <= DEC_MAX_ROWS && P - 1 <= MAX_BEAM;
  // longer prompts: batched passes of up to prefill_rows rows instead of one persistent pass per position
  const bool wide = h->wide_prefill && P - 1 > MAX_BEAM;
  persistent_setup(h, c, prompts, max_new_host, fused ? P : one_pass_prefill || wide ? P - 1 : 0);
  // (capped at 0 new tokens, the prefill and the first step's pass run only for the no-speech probability: they are not
  // decoding steps)
  if (c.max_new > 0 || c.sot != nullptr) {
    // the persistent pass is one cooperative launch per step: no graph needed
    int passes = 0;
    if (fused || one_pass_prefill) {
      const int n = fused ? P : P - 1;
      enqueue_decoder_forward(h, c, fused || ns_in(c, 0, n), n);
      ++passes;
      h->launches += 1;
      ns_reduce(h, c, h->logits.p, [&](int u) { return c.sot[u] < n ? u * n + c.sot[u] : -1; });
    } else if (wide) {
      const int chunk = std::min(P - 1, std::max(1, h->prefill_rows / c.n_utt));
      passes += wide_prefill_ns(h, c, chunk, h->kcache.p, h->vcache.p, static_cast<size_t>(DEC_MAX_ROWS) * T_MAX * h->dims.d_model,
                                T_MAX);
    } else {
      for (int p = 0; p + 1 < P; ++p) {
        enqueue_prefill(h, c, ns_in(c, p, p + 1));
        ++passes;
        h->launches += 2;
        ns_reduce(h, c, h->logits.p, [&](int u) { return c.sot[u] == p ? u * c.beam : -1; });
      }
    }
    if (c.max_new > 0) {
      steps += passes;
      // (fused: step 0 is the search step alone, which is not a pass)
      steps += step_loop(h, c.max_new, true, [&](int gs) {
        if (fused && gs == 0) {
          search_step_run(make_search_args(h, c), h->stream);
          return 2;
        }
        enqueue_step(h, c);
        if (gs == 0) ns_reduce_first_step(h, c, h->logits.p);
        return 1 + 2;  // the pass + the two kernels of the search step
      }) - (fused ? 1 : 0);
    } else if (!fused && ns_in(c, P - 1, P)) {
      enqueue_decoder_forward(h, c, true);  // the first step's pass, without its search
      ++h->launches;
      ns_reduce_first_step(h, c, h->logits.p);
    }
  }
  read_results(h, c, max_new_host, out_ids, out_stride, out_len, out_score);
  return steps;
}


// ------------------------------------------------------------------------------------------------- batched decoder pass
// tile width / split-K of one decoder GEMM for `M` rows: keep >= ~120 CTAs streaming the weight matrix
void plan_dec_gemm(wisb_handle* h, GemmPlan& p, const __half* a, long long lda, const __half* w, int M, int N, int K,
                   GemmEpi e, bool allow_split) {
  const int mt = M / 128;
  int bn = 256;
  while (bn > 64 && (N % bn != 0 || mt * (N / bn) < 120)) bn /= 2;
  int splits = 1;
  if (allow_split) {
    const int kb = K / 64;
    while (mt * (N / bn) * splits < 120 && splits < 8 && kb % (splits * 2) == 0 && kb / (splits * 2) >= 4) splits *= 2;
    e.mode = EPI_F32;
    e.split_stride = static_cast<long long>(M) * N;
  }
  gemm_plan(p, a, lda, w, M, N, K, e, h->num_sms, bn, 0, splits);
}

// layer descriptors + GEMM plans of the batched pass for Rp rows (a multiple of 128): A operands xn / ctx / hid, outputs q
// and the split-K partials `part`; the QKV epilogue writes K/V of row r to slot row_slot[r], position row_pos[r] of
// kc / vc + layer * layer_cache (t_cap positions per slot)
void plan_batch_layers(wisb_handle* h, std::vector<BatchLayer>& layers, int Rp, float* q, __half* xn, __half* ctx,
                       __half* hid, float* part, __half* kc, __half* vc, size_t layer_cache, int t_cap, const int* row_slot,
                       const int* row_pos) {
  const Dims& dm = h->dims;
  const int d = dm.d_model, L = dm.n_dec_layers;
  layers.assign(L, BatchLayer());
  for (int i = 0; i < L; ++i) {
    const DecLayerW& w = h->dec_w[i];
    BatchLayer& b = layers[i];
    b.kcache = kc + layer_cache * i;
    b.vcache = vc + layer_cache * i;
    b.ln1g = w.ln1g; b.ln1b = w.ln1b;
    b.ob = w.ob; b.ln2g = w.ln2g; b.ln2b = w.ln2b;
    b.cob = w.cob; b.ln3g = w.ln3g; b.ln3b = w.ln3b;
    b.fc2b = w.fc2b;
    b.next_g = (i + 1 < L) ? h->dec_w[i + 1].ln1g : h->F("dec.ln.g");
    b.next_b = (i + 1 < L) ? h->dec_w[i + 1].ln1b : h->F("dec.ln.b");
    GemmEpi e;
    e.mode = EPI_DEC_QKV;
    e.bias = w.qkvb;
    e.out = q;
    e.ldo = d;
    e.aux = b.kcache;
    e.aux2 = b.vcache;
    e.d_model = d;
    e.row_slot = row_slot;
    e.row_pos = row_pos;
    e.t_cap = t_cap;
    plan_dec_gemm(h, b.qkv, xn, d, w.qkvw, Rp, 3 * d, d, e, false);
    GemmEpi ep;  // split-K partials; bias / residual / LayerNorm happen in bd_resid_ln_kernel
    ep.out = part;
    ep.ldo = d;
    plan_dec_gemm(h, b.o, ctx, d, w.ow, Rp, d, d, ep, true);
    GemmEpi eq;
    eq.mode = EPI_F32;
    eq.bias = w.cqb;
    eq.out = q;
    eq.ldo = d;
    plan_dec_gemm(h, b.cq, xn, d, w.cqw, Rp, d, d, eq, false);
    plan_dec_gemm(h, b.co, ctx, d, w.cow, Rp, d, d, ep, true);
    GemmEpi e1;
    e1.mode = EPI_F16_GELU;
    e1.bias = w.fc1b;
    e1.out = hid;
    e1.ldo = 4 * d;
    plan_dec_gemm(h, b.fc1, xn, d, w.fc1w, Rp, 4 * d, d, e1, false);
    plan_dec_gemm(h, b.fc2, hid, 4LL * d, w.fc2w, Rp, d, 4 * d, ep, true);
  }
}

// workspaces + GEMM plans of the batched pass for `rows` rows and `t_need` text positions per cache slot
// the row capacity and positions per cache slot ensure_batch(h, rows, t_need) leaves (the workspaces only grow)
int batch_rows_cap(const wisb_handle* h, int rows) { return std::max(round_up(rows, 128), h->bd_rows); }
int batch_tcap(const wisb_handle* h, int t_need) { return std::max(std::min(round_up(t_need, 32), T_MAX), h->bd_tcap); }

void ensure_batch(wisb_handle* h, int rows, int t_need) {
  const Dims& dm = h->dims;
  const int d = dm.d_model, L = dm.n_dec_layers;
  const int Rp = batch_rows_cap(h, rows), tc = batch_tcap(h, t_need);
  // (row tables for every row a pass can carry: a prefill pass has up to the row capacity, more than the search's rows)
  ensure_search(h, Rp);
  // (the QKV epilogues hold the row_slot / row_pos pointers of the search state: a reallocation there stales the plans)
  if (Rp == h->bd_rows && tc == h->bd_tcap && h->bd_search_gen == h->search_gen) return;
  WISB_CUDA(cudaStreamSynchronize(h->stream));
  drop_graphs(h);
  const size_t M = static_cast<size_t>(Rp);
  h->bx.ensure(M * d, true);
  h->bq.ensure(M * d, true);
  h->bxn.ensure(M * d, true);    // rows beyond the live ones stay zero: finite GEMM inputs, outputs never stored
  h->bctx.ensure(M * d, true);
  h->bh.ensure(M * 4 * d, true);
  h->bpart.ensure(8 * M * d, true);
  h->blogits.ensure(M * dm.n_vocab_pad, true);
  const size_t layer_cache = M * tc * d;
  if (layer_cache * L > h->bkc.n) {  // (free first: the two caches are the largest buffers of the handle)
    h->bkc.release();
    h->bvc.release();
  }
  h->bkc.ensure(layer_cache * L, true);
  h->bvc.ensure(layer_cache * L, true);
  plan_batch_layers(h, h->bd_layers, Rp, h->bq.p, h->bxn.p, h->bctx.p, h->bh.p, h->bpart.p, h->bkc.p, h->bvc.p,
                    layer_cache, tc, h->row_slot.p, h->row_pos.p);
  {
    GemmEpi ev;
    ev.mode = EPI_F32;
    ev.out = h->blogits.p;
    ev.ldo = dm.n_vocab_pad;
    plan_dec_gemm(h, h->bd_vocab, h->bxn.p, d, h->H("dec.tok_emb"), Rp, dm.n_vocab_pad, d, ev, false);
  }
  h->bd_rows = Rp;
  h->bd_tcap = tc;
  h->bd_search_gen = h->search_gen;
}

BatchArgs make_batch_args(wisb_handle* h, const DecodeCfg& c) {
  const Dims& dm = h->dims;
  BatchArgs a;
  a.d = dm.d_model;
  a.H = dm.n_heads;
  a.n_utt = c.n_utt;
  a.t_cap = h->bd_tcap;
  a.t_ind = T_MAX;
  a.pdl = h->batch_pdl;
  a.tokens = h->tokens.p;
  a.row_pos = h->row_pos.p;
  a.row_slot = h->row_slot.p;
  a.tok_emb = h->H("dec.tok_emb");
  a.pos_emb = h->F("dec.pos");
  a.x = h->bx.p;
  a.xn = h->bxn.p;
  a.q = h->bq.p;
  a.ctx = h->bctx.p;
  a.part = h->bpart.p;
  a.part_stride = static_cast<long long>(h->bd_rows) * dm.d_model;
  a.indir0 = h->ind0.p;
  a.indir1 = h->ind1.p;
  a.flip = h->flip.p;
  a.vocab = &h->bd_vocab;
  a.cross_tc = h->cross_tc;
  a.num_sms = h->num_sms;
  a.ckv_map = &h->ckv_map;
  a.ckv_base = h->ckv.p;
  if (h->profile) {
    a.prof = [](void* ctx, int cat, int begin) {
      wisb_handle* hh = static_cast<wisb_handle*>(ctx);
      if (begin) hh->prof_begin(cat); else hh->prof_end();
    };
    a.prof_ctx = h;
  }
  return a;
}

SearchArgs make_batch_search_args(wisb_handle* h, const DecodeCfg& c) {
  SearchArgs sa = make_search_args(h, c);
  sa.logits = h->blogits.p;
  return sa;
}

// the pass of one decoding step: n_utt x beam rows at row_pos, K/V into slot row_slot, past positions through indir
BatchArgs batch_step_args(wisb_handle* h, const DecodeCfg& c) {
  BatchArgs a = make_batch_args(h, c);
  a.R = c.n_utt * c.beam;
  a.rows_per_utt = c.beam;
  a.with_logits = 1;
  a.done = h->done.p;
  return a;
}

void enqueue_batch_step(wisb_handle* h, const DecodeCfg& c) {
  BatchArgs a = batch_step_args(h, c);
  h->bd_launches_step = batch_pass_run(a, h->bd_layers.data(), h->dims.n_dec_layers, h->stream) + 2;
  search_step_run(make_batch_search_args(h, c), h->stream);
}

// one batched prefill pass over the row tables prefill_rows_run wrote: chunk positions of each of the c.n_utt windows
BatchArgs batch_prefill_args(wisb_handle* h, const DecodeCfg& c, int chunk, bool with_logits) {
  BatchArgs a = make_batch_args(h, c);
  a.R = c.n_utt * chunk;
  a.rows_per_utt = chunk;
  a.prefill = 1;
  a.with_logits = with_logits ? 1 : 0;
  return a;
}

// Batched prefill: positions [0, n_pos) of the token matrix in h->prompt_dev ([c.n_utt][tok_stride]) as the rows of
// shared passes of at most chunk_max positions per utterance, K/V into cache slot u * slot_stride.  layer_hook(layer,
// chunk), if given, runs after every layer's cross-query GEMM and returns its launches; after_pass(p0, chunk), if given,
// runs after every pass.  A pass yields logits when with_logits, or when logits_if(p0, chunk) says so.  Returns the number
// of passes.
int batch_prefill(wisb_handle* h, const DecodeCfg& c, int tok_stride, int n_pos, int chunk_max, int slot_stride,
                  bool with_logits, const std::function<int(int layer, int chunk)>& layer_hook = nullptr,
                  const std::function<void(int p0, int chunk)>& after_pass = nullptr,
                  const std::function<bool(int p0, int chunk)>& logits_if = nullptr) {
  struct Hook {
    const std::function<int(int, int)>* fn;
    int chunk;
  } hook{&layer_hook, 0};
  int passes = 0;
  for (int p0 = 0; p0 < n_pos; p0 += chunk_max, ++passes) {
    const int chunk = std::min(chunk_max, n_pos - p0);
    prefill_rows_run(h->tokens.p, h->row_pos.p, h->row_slot.p, h->prompt_dev.p, tok_stride, c.n_utt, p0, chunk, slot_stride,
                     h->stream);
    BatchArgs a = batch_prefill_args(h, c, chunk, with_logits || (logits_if && logits_if(p0, chunk)));
    if (layer_hook) {
      hook.chunk = chunk;
      a.layer_hook = [](void* ctx, int layer, cudaStream_t) {
        const Hook* k = static_cast<const Hook*>(ctx);
        return (*k->fn)(layer, k->chunk);
      };
      a.hook_ctx = &hook;
    }
    h->launches += 1 + batch_pass_run(a, h->bd_layers.data(), h->dims.n_dec_layers, h->stream);
    if (after_pass) after_pass(p0, chunk);
  }
  return passes;
}

// workspaces + GEMM plans of the wide prefill passes for `rows` rows, K/V into kc / vc (layer stride layer_cache, t_cap
// positions per slot)
// the row capacity ensure_prefill(h, rows, ...) leaves (the workspaces only grow)
int prefill_rows_cap(const wisb_handle* h, int rows) { return std::max(round_up(rows, 128), h->pf_rows); }

void ensure_prefill(wisb_handle* h, int rows, __half* kc, __half* vc, size_t layer_cache, int t_cap) {
  const int d = h->dims.d_model;
  const int Rp = prefill_rows_cap(h, rows);
  if (Rp == h->pf_rows && kc == h->pf_kc && t_cap == h->pf_tcap && layer_cache == h->pf_layer_cache &&
      !h->pf_layers.empty() && h->pf_layers[0].vcache == vc)
    return;
  WISB_CUDA(cudaStreamSynchronize(h->stream));
  const size_t M = static_cast<size_t>(Rp);
  h->px.ensure(M * d, true);
  h->pq.ensure(M * d, true);
  h->pxn.ensure(M * d, true);  // rows beyond the live ones stay finite: GEMM inputs whose outputs are never stored
  h->pctx.ensure(M * d, true);
  h->ph.ensure(M * 4 * d, true);
  h->ppart.ensure(8 * M * d, true);
  h->ptok.ensure(M, true);
  h->ppos.ensure(M, true);
  h->pslot.ensure(M, true);
  plan_batch_layers(h, h->pf_layers, Rp, h->pq.p, h->pxn.p, h->pctx.p, h->ph.p, h->ppart.p, kc, vc, layer_cache, t_cap,
                    h->pslot.p, h->ppos.p);
  h->pf_rows = Rp;
  h->pf_kc = kc;
  h->pf_tcap = t_cap;
  h->pf_layer_cache = layer_cache;
}

// one wide prefill pass over the row tables prefill_rows_run wrote into ptok / ppos / pslot: ch positions of each of the
// c.n_utt windows, on the wide workspaces and plans ensure_prefill made (t_cap positions per cache slot)
BatchArgs wide_prefill_args(wisb_handle* h, const DecodeCfg& c, int ch, int t_cap) {
  BatchArgs a = make_batch_args(h, c);
  a.R = c.n_utt * ch;
  a.rows_per_utt = ch;
  a.prefill = 1;
  a.wide = 1;
  a.t_cap = t_cap;
  a.tokens = h->ptok.p;
  a.row_pos = h->ppos.p;
  a.row_slot = h->pslot.p;
  a.x = h->px.p;
  a.xn = h->pxn.p;
  a.q = h->pq.p;
  a.ctx = h->pctx.p;
  a.part = h->ppart.p;
  a.part_stride = static_cast<long long>(h->pf_rows) * h->dims.d_model;
  if (h->ckv_is_sw) a.ckv_map = &h->ckv_map_plain;
  return a;
}

// Wide prefill: prompt positions [0, prompt_len - 1) of every utterance in h->prompt_dev as the rows of batched passes of
// `chunk` positions per utterance, K/V into cache slot u * c.beam of kc / vc, cross-attention through
// prefill_cross_attn_launch on h->ckv in the layout the call encoded.  Leaves what the persistent one-pass prefill leaves
// in the cache (the caller then starts the search with the shared-prefix indirection).  after_pass(p0, ch), if given,
// runs after every pass.  Returns the number of passes.
int wide_prefill_run(wisb_handle* h, const DecodeCfg& c, int chunk, __half* kc, __half* vc, size_t layer_cache, int t_cap,
                     const std::function<void(int p0, int ch)>& after_pass = nullptr) {
  const int L = h->dims.n_dec_layers, n_pos = c.prompt_len - 1;
  ensure_prefill(h, c.n_utt * chunk, kc, vc, layer_cache, t_cap);
  for (int i = 0; i < L; ++i) bind_cross_kv(h, h->pf_layers[i], i, c.u0, c.B_total);
  int passes = 0;
  for (int p0 = 0; p0 < n_pos; p0 += chunk, ++passes) {
    const int ch = std::min(chunk, n_pos - p0);
    prefill_rows_run(h->ptok.p, h->ppos.p, h->pslot.p, h->prompt_dev.p, c.prompt_len, c.n_utt, p0, ch, c.beam, h->stream);
    BatchArgs a = wide_prefill_args(h, c, ch, t_cap);
    h->launches += 1 + batch_pass_run(a, h->pf_layers.data(), L, h->stream);
    if (after_pass) after_pass(p0, ch);
  }
  return passes;
}

// the wide prefill passes over positions [0, prompt_len - 1); with the request, every s_u among them is gathered from
// its pass's final-LayerNorm rows into ns_x, and one vocabulary GEMM over ns_x feeds the reduction (a logits buffer for
// every wide-pass row would be n_vocab_pad floats per row: 213 MB at 1024 rows)
int wide_prefill_ns(wisb_handle* h, const DecodeCfg& c, int chunk, __half* kc, __half* vc, size_t layer_cache, int t_cap) {
  const int P = c.prompt_len;
  if (!ns_in(c, 0, P - 1)) return wide_prefill_run(h, c, chunk, kc, vc, layer_cache, t_cap);
  const Dims& dm = h->dims;
  const int cap = round_up(c.n_utt, 128);
  if (cap > h->ns_cap) {
    WISB_CUDA(cudaStreamSynchronize(h->stream));
    h->ns_x.release();
    h->ns_x.ensure(static_cast<size_t>(cap) * dm.d_model, true);  // (rows no window fills stay finite GEMM inputs)
    h->ns_logits.release();
    h->ns_logits.ensure(static_cast<size_t>(cap) * dm.n_vocab_pad);
    GemmEpi e;
    e.mode = EPI_F32;
    e.out = h->ns_logits.p;
    e.ldo = dm.n_vocab_pad;
    plan_dec_gemm(h, h->ns_vocab, h->ns_x.p, dm.d_model, h->H("dec.tok_emb"), cap, dm.n_vocab_pad, dm.d_model, e, false);
    h->ns_cap = cap;
  }
  const int passes = wide_prefill_run(h, c, chunk, kc, vc, layer_cache, t_cap, [&](int p0, int ch) {
    const int* t = ns_table(h, c, [&](int u) { return c.sot[u] >= p0 && c.sot[u] < p0 + ch ? u * ch + c.sot[u] - p0 : -1; });
    if (t == nullptr) return;
    row_gather_run(h->pxn.p, dm.d_model, t, c.n_utt, h->ns_x.p, h->stream);
    ++h->launches;
  });
  gemm_run(h->ns_vocab, h->stream);
  ++h->launches;
  ns_reduce(h, c, h->ns_logits.p, [&](int u) { return c.sot[u] < P - 1 ? u : -1; });
  return passes;
}

// cross K/V of utterance u0 of a batch of B_total encoded windows for every layer of the batched pass
void bind_batch_cross_kv(wisb_handle* h, int u0, int B_total) {
  for (int i = 0; i < h->dims.n_dec_layers; ++i) bind_cross_kv(h, h->bd_layers[i], i, u0, B_total);
}

// decode utterances [u0, u0 + n_utt) of the encoded batch with ONE shared decoder pass per generated token
int decode_batch(wisb_handle* h, const DecodeCfg& c, const int32_t* prompts, const int* max_new_host, int32_t* out_ids,
                 int out_stride, int32_t* out_len, float* out_score) {
  cudaStream_t s = h->stream;
  ensure_batch(h, c.n_utt * c.beam, c.prompt_len + c.max_new);
  bind_batch_cross_kv(h, c.u0, c.B_total);
  int steps = 0;
  upload_prompts(h, prompts, max_new_host, c);
  // (capped at 0 new tokens, the prefill and the first step's pass run only for the no-speech probability: they are not
  // decoding steps)
  if (c.max_new > 0 || c.sot != nullptr) {
    // ---- prompt prefix: every utterance's positions [0, prompt_len - 1) as rows of shared passes (<= 8 positions and
    //      <= the row capacity per pass), K/V into the slot of the utterance's first beam
    const int P = c.prompt_len;
    const int chunk_max = std::max(1, std::min(h->bd_rows / c.n_utt, MAX_BEAM));
    // every prompt position in one pass: that pass also yields the logits of the first step, which then runs no pass
    const bool fused = P <= chunk_max;
    // prompts longer than 9 tokens: wide passes of up to prefill_rows rows (> 8 positions per utterance)
    const int wide = std::min(P - 1, std::max(chunk_max, h->prefill_rows / c.n_utt));
    // utterance u's s_u in the pass of positions [p0, p0 + chunk): its row u * chunk + s_u - p0 of blogits
    auto ns_chunk = [&](int p0, int chunk) {
      ns_reduce(h, c, h->blogits.p, [&](int u) { return c.sot[u] >= p0 && c.sot[u] < p0 + chunk ? u * chunk + c.sot[u] - p0 : -1; });
    };
    int passes;
    if (fused)
      passes = batch_prefill(h, c, P, P, chunk_max, c.beam, true, nullptr, ns_chunk);
    else if (h->wide_prefill && P - 1 > MAX_BEAM && wide > chunk_max)
      passes = wide_prefill_ns(h, c, wide, h->bkc.p, h->bvc.p, static_cast<size_t>(h->bd_rows) * h->bd_tcap * h->dims.d_model,
                               h->bd_tcap);
    else
      passes = batch_prefill(h, c, P, P - 1, chunk_max, c.beam, false, nullptr, ns_chunk,
                             [&](int p0, int chunk) { return ns_in(c, p0, p0 + chunk); });
    search_init_run(make_batch_search_args(h, c), h->prompt_dev.p, s, fused ? P : P - 1);
    if (c.max_new == 0) {
      if (!fused && ns_in(c, P - 1, P)) {  // the first step's pass, without its search
        h->launches += batch_pass_run(batch_step_args(h, c), h->bd_layers.data(), h->dims.n_dec_layers, s);
        ns_reduce_first_step(h, c, h->blogits.p);
      }
      read_results(h, c, max_new_host, out_ids, out_stride, out_len, out_score);
      return steps;
    }
    steps += passes;
    cudaGraphExec_t g = nullptr;
    if (h->use_graphs && !h->profile) {  // (the per-kernel timing hook needs eager launches)
      GraphKey key;
      memset(&key, 0, sizeof(key));
      key.n_utt = c.n_utt; key.beam = c.beam; key.prompt_len = c.prompt_len; key.max_new = c.max_new;
      key.max_hyp = c.mixed ? 0 : c.max_hyp; key.lp = c.mixed ? 0.f : c.lp; key.u0 = c.u0; key.b_total = c.B_total;
      key.mixed = c.mixed;
      key.per_utt_max_new = c.per_utt_max_new;
      key.ts = c.ts; key.ts_max_init = c.ts ? c.ts_max_init : 0;
      key.rep_penalty = c.rep_penalty; key.no_repeat_ngram = c.no_repeat_ngram;
      key.sample = c.sample; key.topk = c.sample ? c.topk : 0; key.temperature = c.sample ? c.temperature : 0.f;
      auto it = h->graphs.find(key);
      if (it == h->graphs.end()) {
        if (h->graphs.size() > 64) drop_graphs(h);
        cudaGraph_t graph;
        cudaGraphExec_t exec;
        WISB_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        enqueue_batch_step(h, c);
        WISB_CUDA(cudaStreamEndCapture(s, &graph));
        WISB_CUDA(cudaGraphInstantiate(&exec, graph, 0));
        WISB_CUDA(cudaGraphDestroy(graph));
        it = h->graphs.emplace(key, exec).first;
      }
      g = it->second;
    }
    // (fused: step 0 is the search step alone, eager, which is not a pass; the graph serves steps >= 1 unchanged)
    steps += step_loop(h, c.max_new, false, [&](int gs) {
      if (fused && gs == 0) {
        search_step_run(make_batch_search_args(h, c), s);
        return 2;
      }
      if (g) WISB_CUDA(cudaGraphLaunch(g, s)); else enqueue_batch_step(h, c);
      if (gs == 0) ns_reduce_first_step(h, c, h->blogits.p);  // (outside the graph: the step graphs stay as they are)
      return h->bd_launches_step;
    }) - (fused ? 1 : 0);
  }
  read_results(h, c, max_new_host, out_ids, out_stride, out_len, out_score);
  return steps;
}

// ------------------------------------------------------------------------------------------------- alignment
// The capture buffer [utterances][A][n_max + 1][F_max] fp32 is the largest workspace of wisb_align (one large-v2 window with
// the default 320 heads, 449 rows and 1500 frames: 0.86 GB): utterances are grouped so that it stays under this cap.
constexpr size_t ALIGN_WS_BYTES = 2ull << 30;

// one group of utterances [g0, g0 + n) whose cross K/V are in h->ckv (encoded as a batch of n): teacher-forced passes with
// the capture hook, token probabilities, filter, DTW, results to the caller's arrays; records the stage events ev[5]
// (passes done), ev[6] (filter done) and ev[7] (DTW done)
void align_group(wisb_handle* h, int g0, int n, const int32_t* start_seq, int S, const int32_t* text, const int32_t* text_len,
                 int text_stride, const int32_t* num_frames, int width, int n_max, int f_max, int32_t* out_path,
                 int path_stride, int32_t* out_path_len, float* out_token_probs, float* cap_out) {
  const Dims& dm = h->dims;
  cudaStream_t s = h->stream;
  const int A = h->al_A;
  int n_grp = 0;
  for (int u = 0; u < n; ++u) n_grp = std::max(n_grp, static_cast<int>(text_len[g0 + u]));
  const int total = S + 1 + n_grp;
  int P = round_up(total, MAX_BEAM);
  if (P > dm.n_text_ctx) P = dm.n_text_ctx;
  ensure_batch(h, n * MAX_BEAM, P);
  bind_batch_cross_kv(h, 0, n);
  // teacher-forced tokens [n][P]: start_seq, <|notimestamps|>, text; rows past an utterance's end feed <|endoftext|>
  // (causal attention keeps the rows before them exact; their outputs are not read)
  const int ts = std::max(text_stride, 1);
  std::vector<int> tok(static_cast<size_t>(n) * P, dm.eot), nt(n), nf(n), txt(static_cast<size_t>(n) * ts, 0);
  for (int u = 0; u < n; ++u) {
    int* t = tok.data() + static_cast<size_t>(u) * P;
    std::copy(start_seq, start_seq + S, t);
    t[S] = dm.no_timestamps;
    nt[u] = text_len[g0 + u];
    nf[u] = num_frames[g0 + u] / 2;
    for (int i = 0; i < nt[u]; ++i) t[S + 1 + i] = txt[static_cast<size_t>(u) * ts + i] = text[static_cast<size_t>(g0 + u) * text_stride + i];
  }
  h->al_ntext.ensure(n);
  h->al_nframes.ensure(n);
  h->al_text.ensure(static_cast<size_t>(n) * ts);
  h->al_cap.ensure(static_cast<size_t>(n) * A * (n_max + 1) * f_max);
  h->al_mat.ensure(static_cast<size_t>(n) * (n_max + 1) * f_max);
  h->al_probs.ensure(static_cast<size_t>(n) * ts);
  h->al_path.ensure(static_cast<size_t>(n) * path_stride * 2);
  h->al_len.ensure(n);
  WISB_CUDA(cudaMemcpyAsync(h->prompt_dev.p, tok.data(), tok.size() * 4, cudaMemcpyHostToDevice, s));
  WISB_CUDA(cudaMemcpyAsync(h->al_ntext.p, nt.data(), n * 4, cudaMemcpyHostToDevice, s));
  WISB_CUDA(cudaMemcpyAsync(h->al_nframes.p, nf.data(), n * 4, cudaMemcpyHostToDevice, s));
  WISB_CUDA(cudaMemcpyAsync(h->al_text.p, txt.data(), txt.size() * 4, cudaMemcpyHostToDevice, s));
  WISB_CUDA(cudaMemsetAsync(h->al_probs.p, 0, static_cast<size_t>(n) * ts * 4, s));
  AlignCaptureArgs cap;  // everything but the layer's cross K, heads and rows per utterance
  cap.head_of = h->al_head.p;
  cap.n_text = h->al_ntext.p;
  cap.n_frames = h->al_nframes.p;
  cap.cap = h->al_cap.p;
  cap.q = h->bq.p;
  cap.row_pos = h->row_pos.p;
  cap.n_utt = n;
  cap.d = dm.d_model;
  cap.H = dm.n_heads;
  cap.A = A;
  cap.s0 = S;
  cap.n_max = n_max;
  cap.f_max = f_max;
  auto capture = [&](int layer, int chunk) {
    const int i0 = h->al_layer_off[layer], i1 = h->al_layer_off[layer + 1];
    if (i0 == i1) return 0;
    AlignCaptureArgs a = cap;
    a.items = h->al_items.p + i0;
    a.n_items = i1 - i0;
    a.ck = h->bd_layers[layer].ck;
    a.rows_per_utt = chunk;
    h->prof_begin(5);
    align_capture_run(a, s);
    h->prof_end();
    return 1;
  };
  auto token_probs = [&](int, int chunk) {
    align_token_probs_run(h->blogits.p, dm.n_vocab_pad, h->row_pos.p, h->al_text.p, ts, h->al_ntext.p, n, chunk, S, dm.eot,
                          h->al_probs.p, s);
    h->launches += 1;
  };
  DecodeCfg c{};
  c.n_utt = n;
  h->timing[6] += static_cast<float>(batch_prefill(h, c, P, P, MAX_BEAM, 1, true, capture, token_probs));
  WISB_CUDA(cudaEventRecord(h->ev[5], s));
  if (cap_out)  // (stream-ordered before the filter standardises the buffer in place)
    WISB_CUDA(cudaMemcpyAsync(cap_out + static_cast<size_t>(g0) * A * (n_max + 1) * f_max, h->al_cap.p,
                              static_cast<size_t>(n) * A * (n_max + 1) * f_max * 4, cudaMemcpyDeviceToHost, s));
  align_filter_run(h->al_cap.p, h->al_mat.p, h->al_ntext.p, h->al_nframes.p, n, A, n_max, f_max, width, s);
  WISB_CUDA(cudaEventRecord(h->ev[6], s));
  align_dtw_run(h->al_mat.p, h->al_ntext.p, h->al_nframes.p, n, n_max, f_max, h->al_path.p, path_stride, h->al_len.p, s);
  WISB_CUDA(cudaEventRecord(h->ev[7], s));
  h->launches += 3;
  WISB_CUDA(cudaMemcpyAsync(out_path + static_cast<size_t>(g0) * path_stride * 2, h->al_path.p,
                            static_cast<size_t>(n) * path_stride * 2 * 4, cudaMemcpyDeviceToHost, s));
  WISB_CUDA(cudaMemcpyAsync(out_path_len + g0, h->al_len.p, n * 4, cudaMemcpyDeviceToHost, s));
  if (text_stride > 0)
    WISB_CUDA(cudaMemcpy2DAsync(out_token_probs + static_cast<size_t>(g0) * text_stride, text_stride * 4, h->al_probs.p, ts * 4,
                                text_stride * 4, n, cudaMemcpyDeviceToHost, s));
  WISB_CUDA(cudaStreamSynchronize(s));
  for (int u = 0; u < n; ++u)
    if (nt[u] == 0) out_path_len[g0 + u] = 0;
}

// entry points without a handle (wisb_buffer_*): the error handling of guarded
template <typename Fn>
int guarded_nohandle(Fn&& fn) {
  try {
    fn();
    return 0;
  } catch (const Error& e) {
    g_last_error = e.what();
    return e.code;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    return 2;
  }
}

// device and size of every live wisb_buffer_alloc allocation (never destroyed: a buffer may be freed during process
// teardown)
std::mutex g_buffer_mu;
std::map<const void*, std::pair<int, size_t>>& buffer_devices() {
  static auto* m = new std::map<const void*, std::pair<int, size_t>>;
  return *m;
}

template <typename Fn>
int guarded(wisb_handle* h, Fn&& fn) {
  try {
    if (h == nullptr) throw Error(1, "null handle");
    std::lock_guard<std::mutex> lock(h->mu);
    WISB_CUDA(cudaSetDevice(h->device));
    fn();
    return 0;
  } catch (const Error& e) {
    g_last_error = e.what();
    if (h && h->stream) {  // leave no dangling capture / sticky state behind
      cudaStreamCaptureStatus cs;
      if (cudaStreamIsCapturing(h->stream, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone) {
        cudaGraph_t g = nullptr;
        cudaStreamEndCapture(h->stream, &g);
        if (g) cudaGraphDestroy(g);
      }
      cudaGetLastError();
    }
    return e.code;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    return 2;
  }
}

int create_common(wisb_handle** out, int device, const std::function<void(wisb_handle*)>& load) {
  if (out == nullptr) {
    g_last_error = "out handle pointer is NULL";
    return 1;
  }
  *out = nullptr;
  std::unique_ptr<wisb_handle> h(new wisb_handle());
  try {
    int n_dev = 0;
    cudaError_t e = cudaGetDeviceCount(&n_dev);
    if (e != cudaSuccess || n_dev == 0)
      throw Error(2, std::string("no CUDA device available (libwisb200 has no CPU fallback): ") + cudaGetErrorString(e));
    WISB_REQUIRE(device >= 0 && device < n_dev, "device index out of range");
    h->device = device;
    WISB_CUDA(cudaSetDevice(device));
    load(h.get());
    finish_create(h.get());
    *out = h.release();
    return 0;
  } catch (const Error& e) {
    g_last_error = e.what();
    return e.code;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    return 2;
  }
}

// `count` elements from the host into a new device buffer (the wisb_debug_dec_* entries)
template <typename T>
T* to_device(DevBuf<T>& d, const void* src, size_t count, cudaStream_t s) {
  d.ensure(count);
  WISB_CUDA(cudaMemcpyAsync(d.p, src, count * sizeof(T), cudaMemcpyHostToDevice, s));
  return d.p;
}

}  // namespace

// ===================================================================================================================== C ABI
extern "C" {

int wisb_abi_version(void) { return WISB_ABI_VERSION; }
const char* wisb_last_error(void) { return g_last_error.c_str(); }

int wisb_create_from_host(const void* blob, size_t nbytes, int device, wisb_handle** out) {
  return create_common(out, device, [&](wisb_handle* h) {
    WISB_REQUIRE(blob != nullptr && nbytes >= 256, "weight blob is NULL or too small");
    h->blob_bytes = nbytes;
    h->own_blob = true;
    WISB_CUDA(cudaMalloc(&h->blob, nbytes));
    WISB_CUDA(cudaMemcpy(h->blob, blob, nbytes, cudaMemcpyHostToDevice));
    const uint8_t* b = static_cast<const uint8_t*>(blob);
    uint32_t n_tensors = 0;
    memcpy(&n_tensors, b + 12, 4);
    const size_t head = 256 + 96ull * n_tensors;
    WISB_REQUIRE(head <= nbytes, "truncated weight blob");
    parse_blob(h, std::vector<uint8_t>(b, b + head));
  });
}

int wisb_create(const char* weights_path, int device, wisb_handle** out) {
  if (weights_path == nullptr) {
    g_last_error = "weights_path is NULL";
    return 1;
  }
  FILE* f = fopen(weights_path, "rb");
  if (!f) {
    g_last_error = std::string("cannot open weight blob '") + weights_path + "'";
    return 1;
  }
  fseek(f, 0, SEEK_END);
  const long long sz = ftell(f);
  fseek(f, 0, SEEK_SET);
  std::vector<uint8_t> buf(static_cast<size_t>(sz > 0 ? sz : 0));
  const size_t got = buf.empty() ? 0 : fread(buf.data(), 1, buf.size(), f);
  fclose(f);
  if (got != buf.size()) {
    g_last_error = "short read on the weight blob";
    return 1;
  }
  return wisb_create_from_host(buf.data(), buf.size(), device, out);
}

int wisb_create_from_device(const void* device_blob, size_t nbytes, int device, wisb_handle** out) {
  return create_common(out, device, [&](wisb_handle* h) {
    WISB_REQUIRE(device_blob != nullptr && nbytes >= 256, "weight blob is NULL or too small");
    h->blob_bytes = nbytes;
    h->own_blob = false;
    h->blob = const_cast<uint8_t*>(static_cast<const uint8_t*>(device_blob));
    std::vector<uint8_t> head(256);
    WISB_CUDA(cudaMemcpy(head.data(), h->blob, 256, cudaMemcpyDeviceToHost));
    uint32_t n_tensors = 0;
    memcpy(&n_tensors, head.data() + 12, 4);
    const size_t hb = 256 + 96ull * n_tensors;
    WISB_REQUIRE(hb <= nbytes, "truncated weight blob");
    head.resize(hb);
    WISB_CUDA(cudaMemcpy(head.data(), h->blob, hb, cudaMemcpyDeviceToHost));
    parse_blob(h, head);
  });
}

int wisb_create_frontend(int device, wisb_handle** out) { return wisb_create_frontend_mels(device, 80, out); }

int wisb_create_frontend_mels(int device, int n_mels, wisb_handle** out) {
  if (n_mels != 80 && n_mels != 128) {
    g_last_error = "n_mels must be 80 or 128";
    return 1;
  }
  return create_common(out, device, [&](wisb_handle* h) { h->dims.n_mels = n_mels; });
}

int wisb_destroy(wisb_handle* h) {
  if (h == nullptr) return 0;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  drop_graphs(h);
  for (auto& e : h->ev)
    if (e) cudaEventDestroy(e);
  for (auto& e : h->prof_ev) cudaEventDestroy(e);
  if (h->own_blob && h->blob) cudaFree(h->blob);
  for (cudaEvent_t ev : h->ev_flag)
    if (ev) cudaEventDestroy(ev);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int wisb_get_dims(wisb_handle* h, int32_t* dims) {
  return guarded(h, [&] {
    WISB_REQUIRE(dims != nullptr, "dims is NULL");
    memcpy(dims, &h->dims, sizeof(Dims));
  });
}

int wisb_set_option(wisb_handle* h, const char* key, int value) {
  return guarded(h, [&] {
    WISB_REQUIRE(key != nullptr, "key is NULL");
    const std::string k(key);
    if (k == "use_graphs") h->use_graphs = value;
    else if (k == "attn_v_mn_major") h->attn_v_mn = value;
    else if (k == "attn_ref") h->attn_ref = value;
    else if (k == "profile") h->profile = value;
    else if (k == "encoder_cache") {
      h->encoder_cache = value ? 1 : 0;
      h->enc_valid = false;
    }
    else if (k == "enc_pdl") h->enc_pdl = value ? 1 : 0;
    else if (k == "batch_rows") {
      WISB_REQUIRE(value >= 8 && value <= 1024, "batch_rows must be in [8, 1024]");
      h->batch_rows = value;
    }
    else if (k == "batch_pdl") h->batch_pdl = value ? 1 : 0;
    else if (k == "debug_chunk") h->debug_chunk = value;
    else if (k == "mega_mma") {  // 1: GEMV phases of the persistent pass on the warp-level tensor path, 0: the SIMT pass
      WISB_REQUIRE(!value || h->mega_img.p != nullptr, "mega_mma needs d_model <= 1280 and a multiple of 64");
      h->mega_mma = value ? 1 : 0;
    }
    else if (k == "cross_tc") {  // 1: wgmma cross-attention in the batched pass, 0: the SIMT cluster kernel (cross-check)
      h->cross_tc = value ? 1 : 0;
      drop_graphs(h);
    }
    else if (k == "decoder_batch") h->decoder_batch = value;  // 2 = use the batched pass even for <= 8 rows (tests)
    else if (k == "wide_prefill") h->wide_prefill = value ? 1 : 0;  // 0: prompts prefill at most 8 positions per pass
    else if (k == "no_speech_prob") h->no_speech = value ? 1 : 0;
    else if (k == "prefill_rows") {
      WISB_REQUIRE(value >= 8 && value <= 65536, "prefill_rows must be in [8, 65536]");
      h->prefill_rows = value;
    }
    else throw Error(1, "unknown option '" + k + "'");
  });
}

int wisb_get_timing(wisb_handle* h, float* out16) {
  return guarded(h, [&] {
    WISB_REQUIRE(out16 != nullptr, "out is NULL");
    memcpy(out16, h->timing, sizeof(h->timing));
  });
}

int wisb_logmel(wisb_handle* h, const void* pcm, int pcm_dtype, int pcm_on_device, const int64_t* offsets,
                const int32_t* n_samples, int B, float* mel_out, int keep_on_device) {
  return guarded(h, [&] {
    WISB_REQUIRE(pcm != nullptr && offsets != nullptr && n_samples != nullptr, "pcm / offsets / n_samples is NULL");
    WISB_REQUIRE(B >= 1 && B <= 4096, "B out of range");
    WISB_REQUIRE(pcm_dtype == WISB_PCM_F32 || pcm_dtype == WISB_PCM_S16, "pcm_dtype must be WISB_PCM_F32 or WISB_PCM_S16");
    const size_t esz = pcm_dtype == WISB_PCM_S16 ? 2 : 4;
    long long total = 0;
    for (int b = 0; b < B; ++b) {
      WISB_REQUIRE(n_samples[b] >= 0 && offsets[b] >= 0, "negative n_samples / offset");
      const long long end = offsets[b] + n_samples[b];
      if (end > total) total = end;
    }
    cudaStream_t s = h->stream;
    ensure_mel(h, B);
    h->pcm_off.ensure(B);
    h->pcm_n.ensure(B);
    WISB_CUDA(cudaEventRecord(h->ev[0], s));
    const void* pcm_d = pcm;
    if (!pcm_on_device) {
      h->pcm_dev.ensure(static_cast<size_t>(total > 0 ? total : 1) * esz);
      if (total > 0) WISB_CUDA(cudaMemcpyAsync(h->pcm_dev.p, pcm, static_cast<size_t>(total) * esz, cudaMemcpyHostToDevice, s));
      pcm_d = h->pcm_dev.p;
    }
    static_assert(sizeof(long long) == sizeof(int64_t), "offset type");
    WISB_CUDA(cudaMemcpyAsync(h->pcm_off.p, offsets, sizeof(int64_t) * B, cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(h->pcm_n.p, n_samples, sizeof(int32_t) * B, cudaMemcpyHostToDevice, s));
    logmel_run(pcm_d, pcm_dtype == WISB_PCM_S16, h->pcm_off.p, h->pcm_n.p, B, h->dims.n_mels, h->lm_tables.p, h->mel.p,
               h->lm_max.p, s);
    if (mel_out != nullptr)
      WISB_CUDA(cudaMemcpyAsync(mel_out, h->mel.p, mel_floats(h, B) * sizeof(float), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaEventRecord(h->ev[1], s));
    WISB_CUDA(cudaStreamSynchronize(s));
    WISB_CUDA(cudaEventElapsedTime(&h->timing[0], h->ev[0], h->ev[1]));
    h->mel_B = keep_on_device ? B : 0;
    if (keep_on_device) h->enc_in_B = 0;  // kept features are now the source of calls with mel == NULL
    h->enc_valid = false;  // the device feature buffer was rewritten
    h->mel_cache_B = 0;
  });
}

int wisb_generate_options_init(wisb_generate_options* opt) {
  return guarded_nohandle([&] {
    WISB_REQUIRE(opt != nullptr, "options pointer is NULL");
    *opt = wisb_generate_options{};
    opt->struct_size = sizeof(wisb_generate_options);
    opt->beam_size = 5;
    opt->patience = 1.f;
    opt->length_penalty = 1.f;
    opt->max_length = 448;
    opt->max_initial_timestamp_index = 50;
    opt->repetition_penalty = 1.f;
    opt->num_hypotheses = 1;
    opt->sampling_topk = 1;
    opt->sampling_temperature = 1.f;
  });
}

int wisb_generate(wisb_handle* h, const float* mel, int B, const int32_t* prompts, int prompt_len,
                  const wisb_generate_options* opt, int32_t* out_ids, int out_stride, int32_t* out_len, float* out_score) {
  return guarded(h, [&] {
    h->ns_B = 0;  // (a failed call leaves no no-speech probabilities to read)
    const Dims& dm = h->dims;
    WISB_REQUIRE(opt != nullptr && opt->struct_size == sizeof(wisb_generate_options),
                 "options are NULL or their struct_size is not sizeof(wisb_generate_options)");
    const wisb_generate_options& o = *opt;
    WISB_REQUIRE(h->blob != nullptr, "handle has no model (created by wisb_create_frontend)");
    WISB_REQUIRE(B >= 1 && B <= 4096, "B out of range");
    WISB_REQUIRE(prompts != nullptr && out_ids != nullptr && out_len != nullptr, "prompts / out_ids / out_len is NULL");
    const bool sample = o.sampling_topk != 1;  // CTranslate2's rule
    const int beam_size = o.beam_size;
    const float patience = sample ? 1.f : o.patience;  // (sampling finishes a window after one hypothesis per row)
    if (o.beam_per_window == nullptr) WISB_REQUIRE(beam_size >= 1 && beam_size <= MAX_BEAM, "beam_size must be in [1, 8]");
    WISB_REQUIRE(prompt_len >= 1 && prompt_len <= dm.n_text_ctx, "prompt length out of range");
    WISB_REQUIRE(o.max_length >= 1 && o.max_length <= dm.n_text_ctx, "max_length must be in [1, n_text_ctx]");
    if (o.patience_per_window == nullptr) WISB_REQUIRE(patience > 0.f, "patience must be positive");
    // hypotheses that finish a window: round half up of beam x patience in fp32, at least 1.  A search records at most
    // beam hypotheses per step over at most 448 steps, so every count above 8 x 448 means "never by count"; clamping
    // at twice that keeps a huge patience from overflowing the int conversion
    auto max_hyp_of = [](int beam, float p) {
      return std::max(1, static_cast<int>(std::min(beam * p + 0.5f, static_cast<float>(2 * MAX_BEAM * T_MAX))));
    };
    // per-window search options: beam, max_hyp and length penalty of every window, and the largest beam (the row block
    // of every window)
    const bool per_window =
        o.beam_per_window != nullptr || o.patience_per_window != nullptr || o.length_penalty_per_window != nullptr;
    if (sample) {
      WISB_REQUIRE(!per_window && beam_size == 1, "sampling: beam_size must be 1, with no per-window search options");
      WISB_REQUIRE(o.num_hypotheses >= 1 && o.num_hypotheses <= MAX_BEAM, "num_hypotheses must be in [1, 8]");
      WISB_REQUIRE(o.sampling_topk == 0 || (o.sampling_topk >= 2 && o.sampling_topk <= MAX_CAND),
                   "sampling_topk must be 0 or in [2, 16]");
      WISB_REQUIRE(std::isfinite(o.sampling_temperature) && o.sampling_temperature > 0.f,
                   "sampling_temperature must be finite and > 0");
      WISB_REQUIRE(o.seeds != nullptr && out_score != nullptr, "seeds / out_score is NULL");
      WISB_REQUIRE(std::isfinite(o.length_penalty), "length_penalty must be finite");
    } else {
      WISB_REQUIRE(o.num_hypotheses == 1, "num_hypotheses must be 1 unless sampling (sampling_topk != 1)");
    }
    std::vector<int> beam_w, hyp_w;
    std::vector<float> lp_w;
    // rows of every window: its beam, or its hypotheses when sampling
    int beam_max = sample ? o.num_hypotheses : beam_size;
    if (per_window) {
      beam_w.resize(B);
      hyp_w.resize(B);
      lp_w.resize(B);
      beam_max = 1;
      for (int b = 0; b < B; ++b) {
        beam_w[b] = o.beam_per_window ? o.beam_per_window[b] : beam_size;
        WISB_REQUIRE(beam_w[b] >= 1 && beam_w[b] <= MAX_BEAM, "per-window beam_size must be in [1, 8]");
        const float p = o.patience_per_window ? o.patience_per_window[b] : patience;
        if (o.patience_per_window) WISB_REQUIRE(std::isfinite(p) && p > 0.f, "per-window patience must be finite and > 0");
        lp_w[b] = o.length_penalty_per_window ? o.length_penalty_per_window[b] : o.length_penalty;
        if (o.length_penalty_per_window) WISB_REQUIRE(std::isfinite(lp_w[b]), "per-window length_penalty must be finite");
        hyp_w[b] = max_hyp_of(beam_w[b], p);
        beam_max = std::max(beam_max, beam_w[b]);
      }
    }
    WISB_REQUIRE(o.n_extra >= 0 && (o.n_extra == 0 || o.extra_suppress != nullptr), "bad extra_suppress");
    for (long long i = 0; i < static_cast<long long>(B) * prompt_len; ++i)
      WISB_REQUIRE(prompts[i] >= 0 && prompts[i] < dm.n_vocab, "prompt token outside the vocabulary");
    WISB_REQUIRE(o.timestamps == 0 || o.timestamps == 1, "timestamps must be 0 or 1");
    WISB_REQUIRE(o.max_initial_timestamp_index >= 0, "max_initial_timestamp_index must be >= 0");
    WISB_REQUIRE(std::isfinite(o.repetition_penalty) && o.repetition_penalty > 0.f,
                 "repetition_penalty must be finite and > 0");
    WISB_REQUIRE(o.no_repeat_ngram_size >= 0 && o.no_repeat_ngram_size <= dm.n_text_ctx,
                 "no_repeat_ngram_size must be in [0, n_text_ctx]");
    if (o.timestamps) {
      WISB_REQUIRE(dm.no_timestamps > dm.eot && dm.no_timestamps + 1 < dm.n_vocab, "this vocabulary has no timestamp tokens");
      // the rules read only generated tokens, so a previous-text context (<|startofprev|> ... before the LAST
      // <|startoftranscript|>) may hold any id, timestamps included; from that sot on (the whole prompt if it has none)
      // <|notimestamps|> and timestamps are refused
      for (int b = 0; b < B; ++b) {
        const int32_t* p = prompts + static_cast<size_t>(b) * prompt_len;
        int from = 0;
        for (int i = 0; i < prompt_len; ++i)
          if (p[i] == dm.sot) from = i;
        for (int i = from; i < prompt_len; ++i) {
          WISB_REQUIRE(p[i] != dm.no_timestamps, "timestamp decoding: the prompt must not contain <|notimestamps|>");
          WISB_REQUIRE(p[i] <= dm.no_timestamps, "timestamp decoding: the prompt must not contain timestamp tokens");
        }
      }
    }
    // the no-speech probability: the position of every window's first <|startoftranscript|> (openai/whisper's sot_index)
    std::vector<int> sot;
    if (h->no_speech) {
      sot.resize(B);
      for (int b = 0; b < B; ++b) {
        const int32_t* p = prompts + static_cast<size_t>(b) * prompt_len;
        sot[b] = static_cast<int>(std::find(p, p + prompt_len, dm.sot) - p);
        WISB_REQUIRE(sot[b] < prompt_len, "no_speech_prob: every prompt must contain <|startoftranscript|>");
      }
      h->ns_prob.ensure(B);
    }
    auto new_tokens = [&](int ml) {  // CTranslate2: at most max_length / 2 new tokens, max_length in total
      int v = ml / 2 < ml - prompt_len ? ml / 2 : ml - prompt_len;
      return v < 0 ? 0 : v;
    };
    int max_new = new_tokens(o.max_length);
    std::vector<int> per_utt;
    if (o.max_length_per_window != nullptr) {
      per_utt.resize(B);
      max_new = 0;
      for (int b = 0; b < B; ++b) {
        WISB_REQUIRE(o.max_length_per_window[b] >= 1 && o.max_length_per_window[b] <= dm.n_text_ctx,
                     "per-utterance max_length out of range");
        per_utt[b] = new_tokens(o.max_length_per_window[b]);
        if (per_utt[b] > max_new) max_new = per_utt[b];
      }
    }
    WISB_REQUIRE(out_stride >= max_new, "out_stride smaller than the maximum number of generated tokens");
    cudaStream_t s = h->stream;
    h->launches = 0;
    for (int i = 1; i <= 5; ++i) h->timing[i] = 0.f;
    WISB_CUDA(cudaEventRecord(h->ev[0], s));
    const bool loaded = loaded_source(h, mel, B);
    const bool cached = !loaded && upload_mel(h, mel, B);
    set_extra_suppress(h, o.extra_suppress, o.n_extra);
    time_h2d(h);
    DecodeCfg c;
    c.prompt_len = prompt_len;
    c.ts = o.timestamps;
    c.ts_max_init = o.max_initial_timestamp_index;
    c.rep_penalty = o.repetition_penalty;
    c.no_repeat_ngram = o.no_repeat_ngram_size;
    // Utterances are encoded and decoded in groups that share every decoder pass: the group's rows (utterances x beams)
    // are the M dimension of the batched pass, so the decoder weights stream once per generated token for the whole
    // group.  The group size only bounds the workspaces (cross K/V: 252 MB per large-v2 utterance).
    const bool persistent = use_persistent_pass(h, B * beam_max);
    int group = persistent ? B : h->batch_rows / beam_max;
    if (group < 1) group = 1;
    int steps = 0;
    for (int g0 = 0; g0 < B; g0 += group) {
      const int n = B - g0 < group ? B - g0 : group;
      encode_stage(h, cached, loaded, B, g0, n, ckv_layout(h, persistent));
      c.u0 = 0;
      c.n_utt = n;
      c.B_total = n;
      // a group whose windows agree on every search option runs the scalar search, else the per-utterance one with
      // the group's largest beam as the row block
      c.beam = beam_size;
      c.max_hyp = max_hyp_of(beam_size, patience);
      c.lp = o.length_penalty;
      c.mixed = 0;
      if (sample) {
        c.beam = o.num_hypotheses;
        c.sample = 1;
        c.topk = o.sampling_topk;
        c.temperature = o.sampling_temperature;
        c.seed_host = o.seeds + g0;
      }
      if (per_window) {
        c.beam = beam_w[g0];
        c.max_hyp = hyp_w[g0];
        c.lp = lp_w[g0];
        for (int u = g0 + 1; u < g0 + n; ++u) {
          if (beam_w[u] != beam_w[g0] || hyp_w[u] != hyp_w[g0] || lp_w[u] != lp_w[g0]) c.mixed = 1;
          c.beam = std::max(c.beam, beam_w[u]);
        }
        c.beam_host = beam_w.data() + g0;
        c.max_hyp_host = hyp_w.data() + g0;
        c.lp_host = lp_w.data() + g0;
      }
      c.max_new = max_new;
      c.per_utt_max_new = 0;
      if (!per_utt.empty()) {
        c.per_utt_max_new = 1;
        c.max_new = 0;
        for (int u = 0; u < n; ++u) c.max_new = per_utt[g0 + u] > c.max_new ? per_utt[g0 + u] : c.max_new;
      }
      if (!sot.empty()) {
        c.sot = sot.data() + g0;
        c.ns_out = h->ns_prob.p + g0;
      }
      ns_begin(h, c);
      const int32_t* gp = prompts + static_cast<size_t>(g0) * prompt_len;
      const int* gmx = per_utt.empty() ? nullptr : per_utt.data() + g0;
      const size_t per = sample ? o.num_hypotheses : 1;  // output entries per window
      int32_t* gi = out_ids + g0 * per * out_stride;
      float* gs = out_score ? out_score + g0 * per : nullptr;
      steps += persistent ? decode_pass(h, c, gp, gmx, gi, out_stride, out_len + g0 * per, gs)
                          : decode_batch(h, c, gp, gmx, gi, out_stride, out_len + g0 * per, gs);
      WISB_CUDA(cudaEventRecord(h->ev[5], s));
      time_group(h, {2, 3, 4});  // encoder, cross K/V, decode
    }
    if (!sot.empty()) {
      h->ns_host.resize(B);
      WISB_CUDA(cudaMemcpyAsync(h->ns_host.data(), h->ns_prob.p, sizeof(float) * B, cudaMemcpyDeviceToHost, s));
      WISB_CUDA(cudaStreamSynchronize(s));
      h->ns_B = B;
    }
    h->timing[6] = static_cast<float>(steps);
    h->timing[7] = static_cast<float>(h->launches);
    h->prof_collect();
  });
}

int wisb_get_no_speech_probs(wisb_handle* h, int B, float* out) {
  return guarded(h, [&] {
    WISB_REQUIRE(out != nullptr, "out is NULL");
    WISB_REQUIRE(h->ns_B > 0, "the last wisb_generate ran without option no_speech_prob, or failed");
    WISB_REQUIRE(B == h->ns_B, "B differs from the last wisb_generate's");
    memcpy(out, h->ns_host.data(), sizeof(float) * B);
  });
}

int wisb_detect_language(wisb_handle* h, const float* mel, int B, int32_t* lang_ids_out, float* probs_out) {
  return guarded(h, [&] {
    const Dims& dm = h->dims;
    WISB_REQUIRE(h->blob != nullptr, "handle has no model (created by wisb_create_frontend)");
    WISB_REQUIRE(B >= 1 && B <= 4096, "B out of range");
    WISB_REQUIRE(lang_ids_out != nullptr && probs_out != nullptr, "output pointer is NULL");
    cudaStream_t s = h->stream;
    const bool loaded = loaded_source(h, mel, B);
    const bool cached = !loaded && upload_mel(h, mel, B);
    encode_stage(h, cached, loaded, B, 0, B, ckv_layout(h, true));  // language detection always runs the persistent pass
    const int nl = dm.n_langs;
    h->lang_ids.ensure(nl);
    std::vector<int> ids(nl);
    for (int i = 0; i < nl; ++i) ids[i] = dm.lang_first + i;
    WISB_CUDA(cudaMemcpyAsync(h->lang_ids.p, ids.data(), sizeof(int) * nl, cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaStreamSynchronize(s));
    const std::vector<int32_t> sot(B, dm.sot);
    for (int u0 = 0; u0 < B; u0 += DEC_MAX_ROWS) {
      DecodeCfg c;
      c.u0 = u0;
      c.n_utt = (B - u0 < DEC_MAX_ROWS) ? B - u0 : DEC_MAX_ROWS;
      c.B_total = B;
      c.beam = 1;
      c.prompt_len = 1;
      c.max_new = 1;
      c.max_hyp = 1;
      c.lp = 1.f;
      persistent_setup(h, c, sot.data(), nullptr);
      enqueue_decoder_forward(h, c, true);
      lang_probs_run(h->logits.p, dm.n_vocab_pad, h->lang_ids.p, nl, c.n_utt, 1, h->lang_probs.p, s);
      WISB_CUDA(cudaMemcpyAsync(h->pin_f.p, h->lang_probs.p, sizeof(float) * c.n_utt * nl, cudaMemcpyDeviceToHost, s));
      WISB_CUDA(cudaStreamSynchronize(s));
      for (int u = 0; u < c.n_utt; ++u) {
        std::vector<int> order(nl);
        for (int i = 0; i < nl; ++i) order[i] = i;
        const float* p = h->pin_f.p + u * nl;
        std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return p[a] > p[b]; });
        for (int i = 0; i < nl; ++i) {
          lang_ids_out[static_cast<size_t>(u0 + u) * nl + i] = ids[order[i]];
          probs_out[static_cast<size_t>(u0 + u) * nl + i] = p[order[i]];
        }
      }
    }
  });
}

int wisb_buffer_alloc(int device, size_t nbytes, void** out) {
  return guarded_nohandle([&] {
    WISB_REQUIRE(out != nullptr, "out is NULL");
    *out = nullptr;
    WISB_REQUIRE(nbytes > 0, "nbytes must be > 0");
    WISB_CUDA(cudaSetDevice(device));
    void* p = nullptr;
    WISB_CUDA(cudaMalloc(&p, nbytes));
    std::lock_guard<std::mutex> lock(g_buffer_mu);
    buffer_devices()[p] = {device, nbytes};
    *out = p;
  });
}

int wisb_buffer_free(void* p) {
  return guarded_nohandle([&] {
    if (p == nullptr) return;
    int device;
    {
      std::lock_guard<std::mutex> lock(g_buffer_mu);
      auto it = buffer_devices().find(p);
      WISB_REQUIRE(it != buffer_devices().end(), "wisb_buffer_free: not a live wisb_buffer_alloc allocation");
      device = it->second.first;
      buffer_devices().erase(it);
    }
    WISB_CUDA(cudaSetDevice(device));
    WISB_CUDA(cudaFree(p));
  });
}

int wisb_buffer_to_host(const void* p, void* host, size_t nbytes) {
  return guarded_nohandle([&] {
    WISB_REQUIRE(host != nullptr || nbytes == 0, "host is NULL");
    int device;
    {
      std::lock_guard<std::mutex> lock(g_buffer_mu);
      auto it = buffer_devices().find(p);
      WISB_REQUIRE(it != buffer_devices().end(), "wisb_buffer_to_host: not a live wisb_buffer_alloc allocation");
      WISB_REQUIRE(nbytes <= it->second.second, "wisb_buffer_to_host: nbytes exceeds the buffer");
      device = it->second.first;
    }
    WISB_CUDA(cudaSetDevice(device));
    if (nbytes) WISB_CUDA(cudaMemcpy(host, p, nbytes, cudaMemcpyDeviceToHost));
  });
}

int wisb_encode(wisb_handle* h, const float* mel, int B, void* out, int out_on_device) {
  return guarded(h, [&] {
    WISB_REQUIRE(h->blob != nullptr, "handle has no model (created by wisb_create_frontend)");
    WISB_REQUIRE(B >= 1 && B <= 4096, "B out of range");
    WISB_REQUIRE(out != nullptr, "out is NULL");
    if (out_on_device) require_on_device(h, out, "out");
    cudaStream_t s = h->stream;
    const size_t row = static_cast<size_t>(h->dims.d_model) * sizeof(__half);
    h->launches = 0;
    for (int i = 1; i <= 5; ++i) h->timing[i] = 0.f;
    WISB_CUDA(cudaEventRecord(h->ev[0], s));
    upload_mel(h, mel, B);
    h->mel_cache_B = 0;  // enc_out is about to hold rows the encoder cache knows nothing of
    time_h2d(h);
    // generate's group at beam 5, so that encoding sizes no workspace beyond what generate would
    const int group = std::max(1, h->batch_rows / 5);
    for (int g0 = 0; g0 < B; g0 += group) {
      const int n = std::min(group, B - g0);
      WISB_CUDA(cudaEventRecord(h->ev[2], s));
      run_encoder(h, n, -1, g0);
      WISB_CUDA(cudaEventRecord(h->ev[3], s));
      // the valid rows only: 1500 of each window's 1536
      WISB_CUDA(cudaMemcpy2DAsync(static_cast<char*>(out) + static_cast<size_t>(g0) * T_ENC * row, T_ENC * row,
                                  h->enc_out.p, T_ENC_PAD * row, T_ENC * row, n, cudaMemcpyDefault, s));
      time_group(h, {2});
    }
    WISB_CUDA(cudaEventRecord(h->ev[4], s));
    WISB_CUDA(cudaStreamSynchronize(s));
    WISB_CUDA(cudaEventElapsedTime(&h->timing[5], h->ev[0], h->ev[4]));
    h->timing[7] = static_cast<float>(h->launches);
    h->prof_collect();
  });
}

int wisb_load_encoder_output(wisb_handle* h, const void* enc, int B, int dtype, int on_device) {
  return guarded(h, [&] {
    WISB_REQUIRE(h->blob != nullptr, "handle has no model (created by wisb_create_frontend)");
    WISB_REQUIRE(B >= 1 && B <= 4096, "B out of range");
    WISB_REQUIRE(enc != nullptr, "enc is NULL");
    WISB_REQUIRE(dtype == 0 || dtype == 1, "dtype must be 0 (float16) or 1 (float32)");
    if (on_device) require_on_device(h, enc, "enc");
    cudaStream_t s = h->stream;
    const size_t n = static_cast<size_t>(B) * T_ENC * h->dims.d_model;
    h->enc_in_B = 0;  // a failure below leaves no half-loaded source behind
    h->enc_in.ensure(n);
    for (int i = 1; i <= 5; ++i) h->timing[i] = 0.f;
    DevBuf<float> staged;  // float32 host input, converted on the device
    WISB_CUDA(cudaEventRecord(h->ev[0], s));
    if (dtype == 0) {
      WISB_CUDA(cudaMemcpyAsync(h->enc_in.p, enc, n * sizeof(__half), on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
    } else if (on_device) {
      f32_to_f16_run(static_cast<const float*>(enc), h->enc_in.p, n, s);
    } else {
      staged.ensure(n);
      WISB_CUDA(cudaMemcpyAsync(staged.p, enc, n * sizeof(float), cudaMemcpyHostToDevice, s));
    }
    WISB_CUDA(cudaEventRecord(h->ev[1], s));
    if (staged.p) f32_to_f16_run(staged.p, h->enc_in.p, n, s);
    WISB_CUDA(cudaStreamSynchronize(s));
    if (!on_device) WISB_CUDA(cudaEventElapsedTime(&h->timing[1], h->ev[0], h->ev[1]));
    h->enc_in_B = B;
    h->mel_B = 0;  // the loaded output, not kept features, is now the source of calls with mel == NULL
  });
}

// --------------------------------------------------------------------------------------------------------------------- diagnostics
int wisb_debug_gemm(wisb_handle* h, const int32_t* prm, int n_prm, const uint16_t* a, const uint16_t* w, const float* bias,
                    const float* pos, const int32_t* row_slot, const int32_t* row_pos, void* out, size_t out_bytes, void* aux,
                    size_t aux_bytes, void* aux2, size_t aux2_bytes, int32_t* plan_out) {
  return guarded(h, [&] {
    WISB_REQUIRE(prm != nullptr && n_prm == 17 && a && w && out, "debug_gemm: bad arguments");
    const int M = prm[0], N = prm[1], K = prm[2], impl = prm[3], bn = prm[4], planner = prm[5], a_wrap = prm[7],
              k_splits = prm[8];
    GemmEpi e;
    e.mode = prm[6];
    e.m_valid = prm[9] > 0 ? prm[9] : M;
    e.n_valid = prm[10] > 0 ? prm[10] : N;
    e.ldo = prm[11] > 0 ? prm[11] : N;
    e.d_model = prm[12];
    e.n_heads = prm[13];
    e.batch = prm[14];
    e.kv_swizzle = prm[15];
    e.t_cap = prm[16];
    WISB_REQUIRE(M > 0 && N > 0 && K > 0 && a_wrap >= 0 && k_splits >= 1 && impl >= 0 && impl <= 1 && planner >= 0 && planner <= 2,
                 "debug_gemm: bad scalar parameters");
    WISB_REQUIRE(e.mode >= EPI_F16 && e.mode <= EPI_DEC_QKV, "debug_gemm: unknown epilogue");
    WISB_REQUIRE(e.m_valid <= M && e.n_valid <= N && e.n_valid % 32 == 0 && e.ldo >= e.n_valid, "debug_gemm: bad m_valid / n_valid / ldo");
    WISB_REQUIRE(planner == 0 || (a_wrap == 0 && k_splits == 1 && bn == 0), "debug_gemm: the decoder planner picks BN and the split itself");
    WISB_REQUIRE(impl == 0 || (e.mode == EPI_F32 && planner == 0 && a_wrap == 0 && k_splits == 1), "debug_gemm: the SIMT check computes plain F32 only");
    cudaStream_t s = h->stream;
    const long long lda = a_wrap > 0 ? a_wrap : K;
    const size_t a_elems = static_cast<size_t>(a_wrap > 0 ? M + 1 : M) * lda;
    DevBuf<__half> da, dw;
    DevBuf<float> dbias, dpos;
    DevBuf<int> dslot, dpos_row;
    DevBuf<uint8_t> dout, daux, daux2;
    da.ensure(a_elems);
    dw.ensure(static_cast<size_t>(N) * K);
    WISB_CUDA(cudaMemcpyAsync(da.p, a, sizeof(__half) * a_elems, cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(dw.p, w, sizeof(__half) * N * K, cudaMemcpyHostToDevice, s));
    if (bias) {
      dbias.ensure(N);
      WISB_CUDA(cudaMemcpyAsync(dbias.p, bias, sizeof(float) * N, cudaMemcpyHostToDevice, s));
      e.bias = dbias.p;
    }
    auto upload = [&](DevBuf<uint8_t>& d, const void* src, size_t bytes) -> void* {
      if (src == nullptr || bytes == 0) return nullptr;
      d.ensure(bytes);
      WISB_CUDA(cudaMemcpyAsync(d.p, src, bytes, cudaMemcpyHostToDevice, s));
      return d.p;
    };
    e.out = upload(dout, out, out_bytes);
    e.aux = upload(daux, aux, aux_bytes);
    e.aux2 = upload(daux2, aux2, aux2_bytes);

    GemmPlan p;
    if (impl == 1) {
      WISB_REQUIRE(out_bytes >= sizeof(float) * M * N, "debug_gemm: out is too small");
      gemm_ref_run(da.p, K, dw.p, static_cast<float*>(e.out), M, N, K, s);
    } else {
      // every address the epilogue can form is checked against the caller's buffers before the launch
      const size_t mv = static_cast<size_t>(e.m_valid), d = static_cast<size_t>(e.d_model), H = static_cast<size_t>(e.n_heads);
      const bool win = e.mode == EPI_CONV2 || e.mode == EPI_CROSSKV || e.mode == EPI_QKV_VT;
      if (e.mode == EPI_CROSSKV || e.mode == EPI_QKV_VT || e.mode == EPI_DEC_QKV)
        WISB_REQUIRE(d > 0 && d % 64 == 0 && (e.mode == EPI_DEC_QKV || H * HEAD_DIM == d), "debug_gemm: d_model / n_heads");
      if (win && e.mode != EPI_CONV2) WISB_REQUIRE(e.batch >= 1 && static_cast<long long>(e.batch) * T_ENC_PAD >= M, "debug_gemm: batch");
      size_t es = 2, need_out = 0, need_aux = 0, need_aux2 = 0;
      switch (e.mode) {
        case EPI_RESID_F32: case EPI_CONV2: case EPI_F32: case EPI_DEC_QKV: es = 4; break;
        default: break;
      }
      need_out = mv * e.ldo * es;
      if (e.mode == EPI_CONV2) {
        WISB_REQUIRE(pos != nullptr, "debug_gemm: CONV2 needs pos");
        dpos.ensure(static_cast<size_t>(T_ENC) * e.ldo);
        WISB_CUDA(cudaMemcpyAsync(dpos.p, pos, sizeof(float) * T_ENC * e.ldo, cudaMemcpyHostToDevice, s));
        e.pos = dpos.p;
      } else if (e.mode == EPI_CROSSKV) {
        WISB_REQUIRE(N % (2 * d) == 0, "debug_gemm: CROSSKV needs N = layers x 2 d_model");
        need_out = static_cast<size_t>(N) * e.batch * T_ENC_PAD * es;
      } else if (e.mode == EPI_QKV_VT) {
        WISB_REQUIRE(N == static_cast<int>(3 * d), "debug_gemm: QKV_VT needs N = 3 d_model");
        need_aux = static_cast<size_t>(e.batch) * d * T_ENC_PAD * 2;
      } else if (e.mode == EPI_DEC_QKV) {
        WISB_REQUIRE(N == static_cast<int>(3 * d) && row_slot && row_pos && e.t_cap > 0, "debug_gemm: DEC_QKV needs N = 3 d_model and rows");
        size_t top = 0;
        for (size_t r = 0; r < mv; ++r) {
          WISB_REQUIRE(row_slot[r] >= 0 && row_pos[r] >= 0 && row_pos[r] < e.t_cap, "debug_gemm: row slot / position out of range");
          const size_t end = (static_cast<size_t>(row_slot[r]) * e.t_cap + row_pos[r] + 1) * d * 2;
          if (end > top) top = end;
        }
        need_aux = need_aux2 = top;
        dslot.ensure(M);
        dpos_row.ensure(M);
        WISB_CUDA(cudaMemcpyAsync(dslot.p, row_slot, sizeof(int) * M, cudaMemcpyHostToDevice, s));
        WISB_CUDA(cudaMemcpyAsync(dpos_row.p, row_pos, sizeof(int) * M, cudaMemcpyHostToDevice, s));
        e.row_slot = dslot.p;
        e.row_pos = dpos_row.p;
      }
      if (planner == 0) {
        if (e.mode == EPI_F32) e.split_stride = static_cast<long long>(M) * e.ldo;
        gemm_plan(p, da.p, lda, dw.p, M, N, K, e, h->num_sms, bn, a_wrap, k_splits);
      } else {
        plan_dec_gemm(h, p, da.p, lda, dw.p, M, N, K, e, planner == 2);
      }
      if (p.epi.mode == EPI_F32) need_out = ((p.k_splits - 1) * static_cast<size_t>(p.epi.split_stride) + mv * e.ldo) * 4;
      WISB_REQUIRE(out_bytes >= need_out && aux_bytes >= need_aux && aux2_bytes >= need_aux2 &&
                       (need_aux == 0 || e.aux != nullptr) && (need_aux2 == 0 || e.aux2 != nullptr),
                   "debug_gemm: an output buffer is too small for the epilogue");
      gemm_run(p, s);
    }
    WISB_CUDA(cudaMemcpyAsync(out, e.out, out_bytes, cudaMemcpyDeviceToHost, s));
    if (e.aux) WISB_CUDA(cudaMemcpyAsync(aux, e.aux, aux_bytes, cudaMemcpyDeviceToHost, s));
    if (e.aux2) WISB_CUDA(cudaMemcpyAsync(aux2, e.aux2, aux2_bytes, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
    if (plan_out) {
      plan_out[0] = impl == 1 ? 0 : p.BN;
      plan_out[1] = impl == 1 ? 0 : p.mcast;
      plan_out[2] = impl == 1 ? 1 : p.k_splits;
      plan_out[3] = impl == 1 ? 0 : p.grid;
    }
  });
}

int wisb_debug_search_step(wisb_handle* h, const int32_t* prm, int n_prm, const float* fprm, int n_fprm,
                           const float* logits, const uint8_t* mask, const int32_t* max_new_u, const int32_t* prompt,
                           const int32_t* beam_u, const int32_t* max_hyp_u, const float* lp_u, const uint64_t* seeds,
                           int32_t* state_i, float* state_f, int32_t* cand_idx, float* cand_score, float* row_lse) {
  return guarded(h, [&] {
    WISB_REQUIRE(prm != nullptr && n_prm == 15 && fprm != nullptr && n_fprm == 3 && logits && mask && state_i && state_f &&
                     cand_idx && cand_score && row_lse,
                 "debug_search_step: bad arguments");
    const int n_utt = prm[0], beam = prm[1], V = prm[2], ldl = prm[3], eot = prm[4], no_ts = prm[5], ts = prm[6];
    const int max_init = prm[7], max_new = prm[8], max_hyp = prm[9], t_max = prm[10], init = prm[11], prompt_len = prm[12];
    WISB_REQUIRE(n_utt >= 1 && beam >= 1 && beam <= MAX_BEAM && n_utt * beam <= 1024 && V >= 2 && V <= TOPK_CHUNKS * 2048 &&
                     ldl >= V && eot >= 0 && eot < V && (ts == 0 || ts == 1) && max_init >= 0 && max_new >= 1 &&
                     max_new <= T_MAX && max_hyp >= 1 && t_max >= 1 && t_max <= T_MAX && init >= 0 && init <= 2,
                 "debug_search_step: bad scalar parameters");
    WISB_REQUIRE(!ts || (no_ts > eot && no_ts + 1 < V && V - no_ts - 1 <= 2048), "debug_search_step: bad timestamp geometry");
    const int no_repeat_ngram = prm[13], topk = prm[14];
    const float length_penalty = fprm[0], rep_penalty = fprm[1], temperature = fprm[2];
    WISB_REQUIRE(std::isfinite(rep_penalty) && rep_penalty > 0.f && no_repeat_ngram >= 0 && no_repeat_ngram <= T_MAX,
                 "debug_search_step: bad history processor arguments");
    const int R = n_utt * beam;
    const bool sample = topk != 1;
    const bool mixed = beam_u != nullptr;
    WISB_REQUIRE(mixed == (max_hyp_u != nullptr) && mixed == (lp_u != nullptr),
                 "debug_search_step: beam_u / max_hyp_u / lp_u come as a set");
    if (sample)
      WISB_REQUIRE(!mixed && seeds != nullptr && (topk == 0 || (topk >= 2 && topk <= MAX_CAND)) &&
                       std::isfinite(temperature) && temperature > 0.f && std::isfinite(length_penalty),
                   "debug_search_step: bad sampling arguments (or per-utterance search options with sampling)");
    // state_i: DecState (5) | flip | seq [2][R][max_new] | indir [2][R][t_max] | tokens [R] | row_pos [R] | done [n_utt] |
    // n_hyp [n_utt] | best_len [H] | best_tokens [H][max_new];  state_f: cum [R] | best_score [H]  (H = n_utt, or R when
    // sampling)
    const int H = sample ? R : n_utt;
    const size_t o_seq = 6, o_ind = o_seq + 2ull * R * max_new, o_tok = o_ind + 2ull * R * t_max, o_rpos = o_tok + R;
    const size_t o_done = o_rpos + R, o_nhyp = o_done + n_utt, o_blen = o_nhyp + n_utt, o_btok = o_blen + H;
    const size_t n_i = o_btok + static_cast<size_t>(H) * max_new, n_f = static_cast<size_t>(R) + H;
    if (init) {
      WISB_REQUIRE(prompt != nullptr && prompt_len >= 1 && prompt_len <= t_max, "debug_search_step: bad prompt");
      for (long long i = 0; i < static_cast<long long>(n_utt) * prompt_len; ++i)
        WISB_REQUIRE(prompt[i] >= 0 && prompt[i] < V, "debug_search_step: prompt token outside the vocabulary");
    } else {
      const int pos = state_i[0], gen = state_i[1], n_done = state_i[2], all_done = state_i[3], flip = state_i[5];
      // (a finished search may sit at gen_step == max_new: its step launches nothing)
      WISB_REQUIRE(pos >= 0 && pos < t_max && gen >= 0 && (gen < max_new || (all_done == 1 && gen == max_new)) &&
                       n_done >= 0 && n_done <= n_utt &&
                       (all_done == 0 || all_done == 1) && state_i[4] == 0 && (flip == 0 || flip == 1),
                   "debug_search_step: bad DecState or flip");
      const int32_t* seq = state_i + o_seq + static_cast<size_t>(flip) * R * max_new;
      const int32_t* ind = state_i + o_ind + static_cast<size_t>(flip) * R * t_max;
      for (int r = 0; r < R; ++r) {
        for (int t = 0; t < gen; ++t)
          WISB_REQUIRE(seq[static_cast<size_t>(r) * max_new + t] >= 0 && seq[static_cast<size_t>(r) * max_new + t] < V,
                       "debug_search_step: history token outside the vocabulary");
        for (int t = 0; t < pos; ++t)
          WISB_REQUIRE(ind[static_cast<size_t>(r) * t_max + t] >= 0 && ind[static_cast<size_t>(r) * t_max + t] < R,
                       "debug_search_step: indirection entry outside [0, R)");
      }
      for (int u = 0; u < n_utt; ++u)
        WISB_REQUIRE(state_i[o_done + u] == 0 || state_i[o_done + u] == 1, "debug_search_step: done must be 0 or 1");
    }
    if (max_new_u)
      for (int u = 0; u < n_utt; ++u)
        WISB_REQUIRE(max_new_u[u] >= 0 && max_new_u[u] <= max_new, "debug_search_step: per-utterance cap outside [0, max_new]");
    if (mixed) {
      for (int u = 0; u < n_utt; ++u)
        WISB_REQUIRE(beam_u[u] >= 1 && beam_u[u] <= beam && max_hyp_u[u] >= 1 && std::isfinite(lp_u[u]),
                     "debug_search_step: per-utterance beam outside [1, beam], max_hyp < 1 or length penalty not finite");
    }
    cudaStream_t s = h->stream;
    DevBuf<float> d_logits, d_lse, d_pmax, d_psum, d_f, d_cs;
    DevBuf<unsigned long long> d_part;
    DevBuf<uint8_t> d_mask;
    DevBuf<int> d_i, d_ci, d_cap, d_prompt, d_slot, d_beam, d_hyp;
    DevBuf<float> d_lp;
    DevBuf<unsigned long long> d_seed;
    d_logits.ensure(static_cast<size_t>(R) * ldl);
    d_mask.ensure(V);
    d_pmax.ensure(static_cast<size_t>(R) * (TOPK_CHUNKS + 1));
    d_psum.ensure(static_cast<size_t>(R) * (TOPK_CHUNKS + 1));
    d_part.ensure(static_cast<size_t>(R) * (TOPK_CHUNKS + 1) * MAX_CAND);
    d_cs.ensure(static_cast<size_t>(n_utt) * MAX_CAND, true);  // (zero when a finished search launches nothing)
    d_ci.ensure(static_cast<size_t>(n_utt) * MAX_CAND, true);
    d_lse.ensure(R, true);
    d_i.ensure(n_i);
    d_f.ensure(n_f);
    d_slot.ensure(R);
    WISB_CUDA(cudaMemcpyAsync(d_logits.p, logits, sizeof(float) * R * ldl, cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(d_mask.p, mask, V, cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(d_i.p, state_i, sizeof(int) * n_i, cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(d_f.p, state_f, sizeof(float) * n_f, cudaMemcpyHostToDevice, s));
    if (max_new_u) {
      d_cap.ensure(n_utt);
      WISB_CUDA(cudaMemcpyAsync(d_cap.p, max_new_u, sizeof(int) * n_utt, cudaMemcpyHostToDevice, s));
    }
    if (mixed) {
      d_beam.ensure(n_utt);
      d_hyp.ensure(n_utt);
      d_lp.ensure(n_utt);
      WISB_CUDA(cudaMemcpyAsync(d_beam.p, beam_u, sizeof(int) * n_utt, cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(d_hyp.p, max_hyp_u, sizeof(int) * n_utt, cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(d_lp.p, lp_u, sizeof(float) * n_utt, cudaMemcpyHostToDevice, s));
    }
    if (sample) {
      d_seed.ensure(n_utt);
      WISB_CUDA(cudaMemcpyAsync(d_seed.p, seeds, sizeof(uint64_t) * n_utt, cudaMemcpyHostToDevice, s));
    }
    if (init) {
      d_prompt.ensure(static_cast<size_t>(n_utt) * prompt_len);
      WISB_CUDA(cudaMemcpyAsync(d_prompt.p, prompt, sizeof(int) * n_utt * prompt_len, cudaMemcpyHostToDevice, s));
    }
    SearchArgs a;
    a.logits = d_logits.p;
    a.ldl = ldl;
    a.n_vocab = V;
    a.mask = d_mask.p;
    a.n_utt = n_utt;
    a.beam = beam;
    a.n_cand = 2 * beam;
    a.max_new = max_new;
    a.max_hyp = max_hyp;
    a.eot = eot;
    a.t_max = t_max;
    a.prompt_len = init ? prompt_len : 1;
    a.length_penalty = length_penalty;
    if (ts) {
      a.ts = 1;
      a.no_ts = no_ts;
      a.ts_begin = no_ts + 1;
      a.ts_max_init = std::min(a.ts_begin + max_init, V - 1);
    }
    a.row_lse = d_lse.p;
    a.part_max = d_pmax.p;
    a.part_sum = d_psum.p;
    a.part = d_part.p;
    a.cand_score = d_cs.p;
    a.cand_idx = d_ci.p;
    a.st = reinterpret_cast<DecState*>(d_i.p);
    a.flip = d_i.p + 5;
    a.seq[0] = d_i.p + o_seq;
    a.seq[1] = d_i.p + o_seq + static_cast<size_t>(R) * max_new;
    a.indir[0] = d_i.p + o_ind;
    a.indir[1] = d_i.p + o_ind + static_cast<size_t>(R) * t_max;
    a.tokens = d_i.p + o_tok;
    a.row_pos = d_i.p + o_rpos;
    a.row_slot = d_slot.p;
    a.done = d_i.p + o_done;
    a.n_hyp = d_i.p + o_nhyp;
    a.best_len = d_i.p + o_blen;
    a.best_tokens = d_i.p + o_btok;
    a.cum = d_f.p;
    a.best_score = d_f.p + R;
    a.max_new_u = max_new_u ? d_cap.p : nullptr;
    a.rep_penalty = rep_penalty;
    a.no_repeat_ngram = no_repeat_ngram;
    if (mixed) {
      a.beam_u = d_beam.p;
      a.max_hyp_u = d_hyp.p;
      a.lp_u = d_lp.p;
    }
    if (sample) {
      a.sample = 1;
      a.topk = topk;
      a.temperature = temperature;
      a.seed_u = d_seed.p;
    }
    static_assert(sizeof(DecState) == 5 * sizeof(int), "DecState is five ints");
    if (init) search_init_run(a, d_prompt.p, s, init == 2 ? prompt_len - 1 : 0);
    search_step_run(a, s);  // the production step: processors, top-k partials, merge, bookkeeping and step advance
    WISB_CUDA(cudaMemcpyAsync(state_i, d_i.p, sizeof(int) * n_i, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(state_f, d_f.p, sizeof(float) * n_f, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(cand_idx, d_ci.p, sizeof(int) * n_utt * MAX_CAND, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(cand_score, d_cs.p, sizeof(float) * n_utt * MAX_CAND, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(row_lse, d_lse.p, sizeof(float) * R, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

// wisb_align's body; cap_out (wisb_debug_align_capture) receives the raw capture buffer [B][A][n_max + 1][F_max]
static void align_impl(wisb_handle* h, const float* mel, int B, const int32_t* start_seq, int start_len, const int32_t* text,
                       const int32_t* text_len, int text_stride, const int32_t* num_frames, int median_filter_width,
                       int32_t* out_path, int path_stride, int32_t* out_path_len, float* out_token_probs, float* cap_out) {
    const Dims& dm = h->dims;
    WISB_REQUIRE(h->blob != nullptr, "handle has no model (created by wisb_create_frontend)");
    WISB_REQUIRE(B >= 1 && B <= 4096, "B out of range");
    WISB_REQUIRE(start_seq != nullptr && text_len != nullptr && num_frames != nullptr && out_path != nullptr &&
                 out_path_len != nullptr && out_token_probs != nullptr, "NULL argument");
    WISB_REQUIRE(start_len >= 1 && start_seq[0] == dm.sot, "start_sequence must begin with <|startoftranscript|>");
    for (int i = 0; i < start_len; ++i)
      WISB_REQUIRE(start_seq[i] >= 0 && start_seq[i] < dm.no_timestamps,
                   "start_sequence must not contain <|notimestamps|> or timestamp tokens");
    WISB_REQUIRE(median_filter_width >= 1 && median_filter_width <= 31 && median_filter_width % 2 == 1,
                 "median_filter_width must be odd and in [1, 31]");
    WISB_REQUIRE(text_stride >= 0 && path_stride >= 0, "negative stride");
    int n_max = 0, f_max = 0;
    for (int b = 0; b < B; ++b) {
      const int n = text_len[b];
      WISB_REQUIRE(n >= 0 && n <= text_stride && (n == 0 || text != nullptr), "text_len out of range");
      WISB_REQUIRE(start_len + 1 + n <= dm.n_text_ctx, "start_sequence + <|notimestamps|> + text exceeds n_text_ctx");
      for (int i = 0; i < n; ++i) {
        const int t = text[static_cast<size_t>(b) * text_stride + i];
        WISB_REQUIRE(t >= 0 && t < dm.eot, "text token outside [0, eot)");
      }
      WISB_REQUIRE(num_frames[b] >= 2 && num_frames[b] <= N_FRAMES, "num_frames must be in [2, 3000]");
      if (n > 0) {
        // a finite matrix gives at most n + F entries; NaN columns (a frame whose probabilities are equal in every row)
        // can route the path along row n to frame 0 and up: n + F + 1
        WISB_REQUIRE(path_stride >= n + num_frames[b] / 2 + 1, "path_stride smaller than len(text) + num_frames // 2 + 1");
        n_max = std::max(n_max, n);
        f_max = std::max(f_max, num_frames[b] / 2);
      }
    }
    for (int b = 0; b < B; ++b) out_path_len[b] = 0;
    if (text_stride > 0) std::fill(out_token_probs, out_token_probs + static_cast<size_t>(B) * text_stride, 0.f);
    for (int i = 1; i <= 7; ++i) h->timing[i] = 0.f;
    h->timing[13] = h->timing[14] = 0.f;
    if (n_max == 0) return;  // no text anywhere: nothing to align
    cudaStream_t s = h->stream;
    h->launches = 0;
    WISB_CUDA(cudaEventRecord(h->ev[0], s));
    const bool loaded = loaded_source(h, mel, B);
    const bool cached = !loaded && upload_mel(h, mel, B);
    time_h2d(h);
    const size_t per_utt = static_cast<size_t>(h->al_A) * (n_max + 1) * f_max * sizeof(float);
    int group = std::min(h->batch_rows / MAX_BEAM, static_cast<int>(std::min<size_t>(ALIGN_WS_BYTES / per_utt, 4096)));
    if (group < 1) group = 1;
    for (int g0 = 0; g0 < B; g0 += group) {
      const int n = std::min(group, B - g0);
      encode_stage(h, cached, loaded, B, g0, n, ckv_layout(h, false));  // the capture and the batched pass read linear cross K/V
      align_group(h, g0, n, start_seq, start_len, text, text_len, text_stride, num_frames, median_filter_width, n_max, f_max,
                  out_path, path_stride, out_path_len, out_token_probs, cap_out);
      time_group(h, {2, 2, 3, 4, 14});  // encoder + cross K/V, passes, filter, DTW
    }
    h->timing[7] = static_cast<float>(h->launches);
    const float dtw = h->timing[14];
    h->prof_collect();  // (capture kernels are profile category 5 -> timing[13])
    h->timing[14] = dtw;
}

int wisb_align(wisb_handle* h, const float* mel, int B, const int32_t* start_seq, int start_len, const int32_t* text,
               const int32_t* text_len, int text_stride, const int32_t* num_frames, int median_filter_width,
               int32_t* out_path, int path_stride, int32_t* out_path_len, float* out_token_probs) {
  return guarded(h, [&] {
    align_impl(h, mel, B, start_seq, start_len, text, text_len, text_stride, num_frames, median_filter_width, out_path,
               path_stride, out_path_len, out_token_probs, nullptr);
  });
}

int wisb_debug_align_capture(wisb_handle* h, const float* mel, int B, const int32_t* start_seq, int start_len,
                             const int32_t* text, const int32_t* text_len, int text_stride, const int32_t* num_frames,
                             float* cap_out) {
  return guarded(h, [&] {
    WISB_REQUIRE(cap_out != nullptr && text_len != nullptr && num_frames != nullptr && B >= 1 && B <= 4096, "bad arguments");
    int stride = 1;
    for (int b = 0; b < B; ++b) stride = std::max(stride, text_len[b] + num_frames[b] / 2 + 1);
    std::vector<int32_t> path(static_cast<size_t>(B) * stride * 2), len(B);
    std::vector<float> probs(static_cast<size_t>(B) * std::max(text_stride, 1));
    align_impl(h, mel, B, start_seq, start_len, text, text_len, text_stride, num_frames, 7, path.data(), stride, len.data(),
               probs.data(), cap_out);
  });
}

int wisb_debug_align_post(wisb_handle* h, const float* weights, int A, int R, int F, int width, int dtw_only,
                          float* matrix_out, int32_t* path_out, int32_t* path_len) {
  return guarded(h, [&] {
    WISB_REQUIRE(weights != nullptr && path_out != nullptr && path_len != nullptr, "NULL argument");
    WISB_REQUIRE(R >= 2 && R <= T_MAX + 1 && F >= 1 && F <= T_ENC && A >= 1 && A <= 4096, "debug_align_post: bad shape");
    WISB_REQUIRE(!dtw_only || A == 1, "debug_align_post: dtw_only takes one matrix (A = 1)");
    WISB_REQUIRE(dtw_only || (width >= 1 && width <= 31 && width % 2 == 1), "median filter width must be odd and in [1, 31]");
    cudaStream_t s = h->stream;
    const size_t cells = static_cast<size_t>(R) * F;
    DevBuf<float> cap, mat;
    DevBuf<int> meta, path;
    mat.ensure(cells);
    meta.ensure(3);
    path.ensure(static_cast<size_t>(R + F) * 2, true);
    const int nt_nf[2] = {R - 1, F};
    WISB_CUDA(cudaMemcpyAsync(meta.p, nt_nf, sizeof(nt_nf), cudaMemcpyHostToDevice, s));
    if (dtw_only) {
      WISB_CUDA(cudaMemcpyAsync(mat.p, weights, cells * 4, cudaMemcpyHostToDevice, s));
    } else {
      cap.ensure(cells * A);
      WISB_CUDA(cudaMemcpyAsync(cap.p, weights, cells * A * 4, cudaMemcpyHostToDevice, s));
      align_filter_run(cap.p, mat.p, meta.p, meta.p + 1, 1, A, R - 1, F, width, s);
    }
    align_dtw_run(mat.p, meta.p, meta.p + 1, 1, R - 1, F, path.p, R + F, meta.p + 2, s);
    if (matrix_out) WISB_CUDA(cudaMemcpyAsync(matrix_out, mat.p, cells * 4, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(path_out, path.p, static_cast<size_t>(R + F) * 2 * 4, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(path_len, meta.p + 2, 4, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_no_speech_probs(wisb_handle* h, const float* logits, int n_rows, int ldl, const int32_t* rows, int n,
                               int n_vocab, int no_speech, float* out) {
  return guarded(h, [&] {
    WISB_REQUIRE(logits && rows && out, "debug_no_speech_probs: NULL argument");
    WISB_REQUIRE(n_rows >= 1 && n >= 1 && n <= 65535 && n_vocab >= 1 && ldl >= n_vocab && no_speech >= 0 && no_speech < n_vocab,
                 "debug_no_speech_probs: bad geometry");
    for (int u = 0; u < n; ++u) WISB_REQUIRE(rows[u] < n_rows, "debug_no_speech_probs: row index out of range");
    cudaStream_t s = h->stream;
    DevBuf<float> dl, dout;
    DevBuf<int> drows;
    dl.ensure(static_cast<size_t>(n_rows) * ldl);
    dout.ensure(n);
    drows.ensure(n);
    WISB_CUDA(cudaMemcpyAsync(dl.p, logits, sizeof(float) * n_rows * static_cast<size_t>(ldl), cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(drows.p, rows, sizeof(int) * n, cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(dout.p, out, sizeof(float) * n, cudaMemcpyHostToDevice, s));
    no_speech_run(dl.p, ldl, drows.p, n, n_vocab, no_speech, dout.p, s);
    WISB_CUDA(cudaMemcpyAsync(out, dout.p, sizeof(float) * n, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_enc_attn(wisb_handle* h, const uint16_t* qkv16, int B, int d, int H, int impl, uint16_t* ctx16_out) {
  return guarded(h, [&] {
    WISB_REQUIRE(qkv16 && ctx16_out && B >= 1 && H >= 1 && d == H * HEAD_DIM && impl >= 0 && impl <= 2, "debug_enc_attn: bad arguments");
    cudaStream_t s = h->stream;
    const size_t rows = static_cast<size_t>(B) * T_ENC_PAD;
    DevBuf<__half> dq, dvt, dctx;
    dq.ensure(rows * 3 * d);
    dctx.ensure(rows * d, true);
    WISB_CUDA(cudaMemcpyAsync(dq.p, qkv16, sizeof(__half) * rows * 3 * d, cudaMemcpyHostToDevice, s));
    if (impl == 2) {
      enc_attn_ref_run(dq.p, dctx.p, B, d, H, s);
    } else {
      if (impl == 1) {  // the layout EPI_QKV_VT writes: vt[((b H + head) 64 + e) 1536 + t] = V[b 1536 + t][head 64 + e]
        std::vector<uint16_t> vt(rows * d);
        for (size_t r = 0; r < rows; ++r) {
          const size_t b = r / T_ENC_PAD, t = r % T_ENC_PAD;
          for (int c = 0; c < d; ++c) vt[((b * H + c / HEAD_DIM) * HEAD_DIM + c % HEAD_DIM) * T_ENC_PAD + t] = qkv16[r * 3 * d + 2 * d + c];
        }
        dvt.ensure(rows * d);
        WISB_CUDA(cudaMemcpyAsync(dvt.p, vt.data(), sizeof(__half) * rows * d, cudaMemcpyHostToDevice, s));
        WISB_CUDA(cudaStreamSynchronize(s));  // (vt is a host temporary)
      }
      AttnPlan ap;
      enc_attn_plan(ap, dq.p, dvt.p, dctx.p, B, d, H, impl == 0);
      enc_attn_run(ap, s);
    }
    WISB_CUDA(cudaMemcpyAsync(ctx16_out, dctx.p, sizeof(__half) * rows * d, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

// The batched decoder pass's own kernels on caller data, through the launchers batch_pass_run uses (decoder.cuh), without
// programmatic dependent launch.  Every index a kernel can form is checked against the caller's sizes first.
int wisb_debug_dec_cross_attn(wisb_handle* h, const int32_t* prm, int n_prm, const float* q, const uint16_t* ckv,
                              const int32_t* done, uint16_t* ctx16) {
  return guarded(h, [&] {
    WISB_REQUIRE(prm != nullptr && n_prm == 6 && q && ckv && ctx16, "debug_dec_cross_attn: bad arguments");
    const int n_utt = prm[0], rpu = prm[1], H = prm[2], n_layers = prm[3], layer = prm[4], impl = prm[5];
    WISB_REQUIRE(n_utt >= 1 && n_utt <= BD_CROSS_MAX_UTT,
                 "debug_dec_cross_attn: 1.." + std::to_string(BD_CROSS_MAX_UTT) + " utterances in one pass");
    WISB_REQUIRE(rpu >= 1 && rpu <= MAX_BEAM, "debug_dec_cross_attn: 1..8 rows per utterance");
    WISB_REQUIRE(H >= 1 && H <= 32 && n_layers >= 1 && layer >= 0 && layer < n_layers && (impl == 0 || impl == 1),
                 "debug_dec_cross_attn: bad heads / layer / impl");
    cudaStream_t s = h->stream;
    const int d = H * HEAD_DIM;
    const size_t rows = static_cast<size_t>(n_utt) * rpu;
    const size_t block = static_cast<size_t>(n_utt) * H * T_ENC_PAD * HEAD_DIM;  // one layer's K (or V), all utterances
    const size_t ckv_elems = static_cast<size_t>(n_layers) * 2 * block;
    DevBuf<float> dq;
    DevBuf<__half> dckv, dctx;
    DevBuf<int> ddone;
    BatchArgs a;
    a.R = static_cast<int>(rows);
    a.d = d;
    a.H = H;
    a.n_utt = n_utt;
    a.rows_per_utt = rpu;
    a.q = to_device(dq, q, rows * d, s);
    a.ctx = to_device(dctx, ctx16, rows * d, s);
    a.done = done ? to_device(ddone, done, n_utt, s) : nullptr;
    a.cross_tc = impl == 0 ? 1 : 0;
    a.num_sms = h->num_sms;
    a.ckv_base = to_device(dckv, ckv, ckv_elems, s);
    CUtensorMap map;  // as the engine's ckv_map: the whole buffer as rows of one head's 64 values
    make_tmap_f16_2d(&map, dckv.p, HEAD_DIM, static_cast<long long>(ckv_elems / HEAD_DIM), HEAD_DIM, HEAD_DIM, 128);
    a.ckv_map = &map;
    BatchLayer ly;
    ly.ck = dckv.p + static_cast<size_t>(2 * layer) * block;
    ly.cv = dckv.p + static_cast<size_t>(2 * layer + 1) * block;
    cross_attn_launch(a, ly, s);
    WISB_CUDA(cudaMemcpyAsync(ctx16, dctx.p, sizeof(__half) * rows * d, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_dec_prefill_cross_attn(wisb_handle* h, const int32_t* prm, int n_prm, const float* q, const uint16_t* ckv,
                                      uint16_t* ctx16) {
  return guarded(h, [&] {
    WISB_REQUIRE(prm != nullptr && n_prm == 6 && q && ckv && ctx16, "debug_dec_prefill_cross_attn: bad arguments");
    const int n_utt = prm[0], rpu = prm[1], H = prm[2], n_layers = prm[3], layer = prm[4], swizzled = prm[5];
    WISB_REQUIRE(n_utt >= 1 && n_utt <= BD_CROSS_MAX_UTT,
                 "debug_dec_prefill_cross_attn: 1.." + std::to_string(BD_CROSS_MAX_UTT) + " utterances in one pass");
    WISB_REQUIRE(rpu >= 1 && rpu <= T_MAX, "debug_dec_prefill_cross_attn: 1..448 rows per utterance");
    WISB_REQUIRE(H >= 1 && H <= 32 && n_layers >= 1 && layer >= 0 && layer < n_layers && (swizzled == 0 || swizzled == 1),
                 "debug_dec_prefill_cross_attn: bad heads / layer / swizzled");
    cudaStream_t s = h->stream;
    const int d = H * HEAD_DIM;
    const size_t rows = static_cast<size_t>(n_utt) * rpu;
    const size_t block = static_cast<size_t>(n_utt) * H * T_ENC_PAD * HEAD_DIM;  // one layer's K (or V), all utterances
    const size_t ckv_elems = static_cast<size_t>(n_layers) * 2 * block;
    WISB_REQUIRE(ckv_elems / HEAD_DIM < (1ull << 31), "debug_dec_prefill_cross_attn: cross K/V too large for one tensor map");
    DevBuf<float> dq;
    DevBuf<__half> dckv, dctx;
    BatchArgs a;
    a.R = static_cast<int>(rows);
    a.d = d;
    a.H = H;
    a.n_utt = n_utt;
    a.rows_per_utt = rpu;
    a.prefill = 1;
    a.wide = 1;
    a.q = to_device(dq, q, rows * d, s);
    a.ctx = to_device(dctx, ctx16, rows * d, s);
    a.num_sms = h->num_sms;
    a.ckv_base = to_device(dckv, ckv, ckv_elems, s);
    CUtensorMap map;  // as the engine's ckv_map (linear layout) or ckv_map_plain (chunk-swizzled layout)
    make_tmap_f16_2d_swizzle(&map, dckv.p, HEAD_DIM, static_cast<long long>(ckv_elems / HEAD_DIM), HEAD_DIM, HEAD_DIM, 128,
                             swizzled == 0);
    a.ckv_map = &map;
    BatchLayer ly;
    ly.ck = dckv.p + static_cast<size_t>(2 * layer) * block;
    ly.cv = dckv.p + static_cast<size_t>(2 * layer + 1) * block;
    prefill_cross_attn_launch(a, ly, s);
    WISB_CUDA(cudaMemcpyAsync(ctx16, dctx.p, sizeof(__half) * rows * d, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_dec_self_attn(wisb_handle* h, const int32_t* prm, int n_prm, const float* q, const uint16_t* kcache,
                             const uint16_t* vcache, const int32_t* row_pos, const int32_t* row_slot, const int32_t* indir0,
                             const int32_t* indir1, const int32_t* done, uint16_t* ctx16) {
  return guarded(h, [&] {
    WISB_REQUIRE(prm != nullptr && n_prm == 8 && q && kcache && vcache && row_pos && row_slot && indir0 && indir1 && ctx16,
                 "debug_dec_self_attn: bad arguments");
    const int R = prm[0], H = prm[1], n_slots = prm[2], t_cap = prm[3], t_ind = prm[4], rpu = prm[5], prefill = prm[6],
              flip = prm[7];
    WISB_REQUIRE(rpu >= 1 && rpu <= MAX_BEAM && R >= 1 && R <= 65535 && R % rpu == 0,
                 "debug_dec_self_attn: R = utterances x 1..8 rows per utterance");
    WISB_REQUIRE(H >= 1 && H <= 32 && n_slots >= 1 && t_cap >= 1 && t_ind >= 1 && t_ind <= T_MAX,
                 "debug_dec_self_attn: bad heads / slots / t_cap / t_ind (<= 448)");
    WISB_REQUIRE((prefill == 0 || prefill == 1) && (flip == 0 || flip == 1), "debug_dec_self_attn: prefill and flip are 0 / 1");
    for (int r = 0; r < R; ++r)
      WISB_REQUIRE(row_slot[r] >= 0 && row_slot[r] < n_slots && row_pos[r] >= 0 && row_pos[r] < t_cap && row_pos[r] < t_ind,
                   "debug_dec_self_attn: row slot / position out of range");
    const size_t n_ind = static_cast<size_t>(R) * t_ind;
    for (size_t i = 0; i < n_ind; ++i)
      WISB_REQUIRE(indir0[i] >= 0 && indir0[i] < n_slots && indir1[i] >= 0 && indir1[i] < n_slots,
                   "debug_dec_self_attn: indirection entry out of range");
    cudaStream_t s = h->stream;
    const int d = H * HEAD_DIM;
    const size_t cache = static_cast<size_t>(n_slots) * t_cap * d;
    DevBuf<float> dq;
    DevBuf<__half> dk, dv, dctx;
    DevBuf<int> dpos, dslot, di0, di1, dflip, ddone;
    BatchArgs a;
    a.R = R;
    a.d = d;
    a.H = H;
    a.n_utt = R / rpu;
    a.rows_per_utt = rpu;
    a.t_cap = t_cap;
    a.t_ind = t_ind;
    a.prefill = prefill;
    a.q = to_device(dq, q, static_cast<size_t>(R) * d, s);
    a.ctx = to_device(dctx, ctx16, static_cast<size_t>(R) * d, s);
    a.row_pos = to_device(dpos, row_pos, R, s);
    a.row_slot = to_device(dslot, row_slot, R, s);
    a.indir0 = to_device(di0, indir0, n_ind, s);
    a.indir1 = to_device(di1, indir1, n_ind, s);
    a.flip = to_device(dflip, &flip, 1, s);
    a.done = done ? to_device(ddone, done, R / rpu, s) : nullptr;
    BatchLayer ly;
    ly.kcache = to_device(dk, kcache, cache, s);
    ly.vcache = to_device(dv, vcache, cache, s);
    self_attn_launch(a, ly, s);
    WISB_CUDA(cudaMemcpyAsync(ctx16, dctx.p, sizeof(__half) * R * d, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_dec_resid_ln(wisb_handle* h, int R, int cap, int d, int n_splits, int64_t split_stride, const float* part,
                            size_t part_elems, const float* bias, const float* g, const float* b, float* x, uint16_t* xn16) {
  return guarded(h, [&] {
    WISB_REQUIRE(part && bias && g && b && x && xn16, "debug_dec_resid_ln: NULL argument");
    WISB_REQUIRE(R >= 1 && cap >= R && d >= 128 && d % 128 == 0 && d <= 1536, "debug_dec_resid_ln: d_model multiple of 128, <= 1536");
    WISB_REQUIRE(n_splits == 1 || n_splits == 2 || n_splits == 4 || n_splits == 8, "debug_dec_resid_ln: 1, 2, 4 or 8 slabs");
    const size_t rd = static_cast<size_t>(R) * d, cd = static_cast<size_t>(cap) * d;
    WISB_REQUIRE(split_stride % 4 == 0 && (n_splits == 1 || split_stride >= static_cast<int64_t>(rd)) &&
                     part_elems >= static_cast<size_t>(n_splits - 1) * static_cast<size_t>(split_stride) + rd,
                 "debug_dec_resid_ln: slabs overlap, are misaligned or exceed the partial buffer");
    cudaStream_t s = h->stream;
    DevBuf<float> dx, dpart, dbias, dg, db;
    DevBuf<__half> dxn;
    BatchArgs a;
    a.R = R;
    a.d = d;
    a.x = to_device(dx, x, cd, s);
    a.xn = to_device(dxn, xn16, cd, s);
    a.part = to_device(dpart, part, part_elems, s);
    a.part_stride = split_stride;
    resid_ln_launch(a, n_splits, to_device(dbias, bias, d, s), to_device(dg, g, d, s), to_device(db, b, d, s), s);
    WISB_CUDA(cudaMemcpyAsync(x, dx.p, sizeof(float) * cd, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(xn16, dxn.p, sizeof(__half) * cd, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_dec_embed_ln(wisb_handle* h, int R, int cap, int d, int n_vocab, int n_pos, const int32_t* tokens, const int32_t* row_pos,
                            const uint16_t* tok_emb, const float* pos_emb, const float* g, const float* b, float* x,
                            uint16_t* xn16) {
  return guarded(h, [&] {
    WISB_REQUIRE(tokens && row_pos && tok_emb && pos_emb && g && b && x && xn16, "debug_dec_embed_ln: NULL argument");
    WISB_REQUIRE(R >= 1 && cap >= R && d >= 128 && d % 128 == 0 && d <= 1536, "debug_dec_embed_ln: d_model multiple of 128, <= 1536");
    WISB_REQUIRE(n_vocab >= 1 && n_pos >= 1, "debug_dec_embed_ln: empty embedding table");
    for (int r = 0; r < R; ++r)
      WISB_REQUIRE(tokens[r] >= 0 && tokens[r] < n_vocab && row_pos[r] >= 0 && row_pos[r] < n_pos,
                   "debug_dec_embed_ln: token / position out of range");
    cudaStream_t s = h->stream;
    const size_t cd = static_cast<size_t>(cap) * d;
    DevBuf<float> dx, dpos, dg, db;
    DevBuf<__half> dxn, demb;
    DevBuf<int> dtok, drow;
    BatchArgs a;
    a.R = R;
    a.d = d;
    a.tokens = to_device(dtok, tokens, R, s);
    a.row_pos = to_device(drow, row_pos, R, s);
    a.tok_emb = to_device(demb, tok_emb, static_cast<size_t>(n_vocab) * d, s);
    a.pos_emb = to_device(dpos, pos_emb, static_cast<size_t>(n_pos) * d, s);
    a.x = to_device(dx, x, cd, s);
    a.xn = to_device(dxn, xn16, cd, s);
    embed_ln_launch(a, to_device(dg, g, d, s), to_device(db, b, d, s), s);
    WISB_CUDA(cudaMemcpyAsync(x, dx.p, sizeof(float) * cd, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(xn16, dxn.p, sizeof(__half) * cd, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_encode(wisb_handle* h, const float* mel, int B, float* enc_out, int n_layers) {
  return guarded(h, [&] {
    WISB_REQUIRE(h->blob != nullptr && enc_out != nullptr && B >= 1, "bad arguments");
    const int d = h->dims.d_model;
    cudaStream_t s = h->stream;
    upload_mel(h, mel, B);
    run_encoder(h, B, n_layers);
    std::vector<__half> tmp(static_cast<size_t>(B) * T_ENC_PAD * d);
    WISB_CUDA(cudaMemcpyAsync(tmp.data(), h->enc_out.p, tmp.size() * sizeof(__half), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
    for (int b = 0; b < B; ++b)
      for (int t = 0; t < T_ENC; ++t)
        for (int e = 0; e < d; ++e)
          enc_out[(static_cast<size_t>(b) * T_ENC + t) * d + e] = __half2float(tmp[(static_cast<size_t>(b) * T_ENC_PAD + t) * d + e]);
  });
}

int wisb_debug_enc_stem(wisb_handle* h, const float* mel, int B, uint16_t* h1_out, float* x_out) {
  return guarded(h, [&] {
    WISB_REQUIRE(h->blob != nullptr && mel && h1_out && x_out, "debug_enc_stem: bad arguments");
    WISB_REQUIRE(B >= 1 && B <= 4096, "debug_enc_stem: B out of range");
    const int d = h->dims.d_model;
    cudaStream_t s = h->stream;
    upload_mel(h, mel, B);
    ensure_encoder(h, B);
    h->enc_valid = false;
    h->mel_cache_B = 0;
    enc_stem_run(h, B, 0);
    const size_t n1 = (static_cast<size_t>(B) * H1_ROWS + 8) * d, nx = static_cast<size_t>(B) * T_ENC_PAD * d;
    WISB_CUDA(cudaMemcpyAsync(h1_out, h->h1.p, n1 * sizeof(__half), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(x_out, h->x.p, nx * sizeof(float), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_enc_ln(wisb_handle* h, const float* x, int rows, int d, const float* g, const float* b, int pdl, uint16_t* y) {
  return guarded(h, [&] {
    WISB_REQUIRE(x && g && b && y, "debug_enc_ln: NULL argument");
    WISB_REQUIRE(rows >= 1 && rows <= 4096 * T_ENC_PAD, "debug_enc_ln: rows out of range");
    WISB_REQUIRE(d >= 128 && d % 128 == 0 && d <= 1536 && (pdl == 0 || pdl == 1),
                 "debug_enc_ln: d_model a multiple of 128, <= 1536; pdl 0 / 1");
    h->enc_valid = false;
    cudaStream_t s = h->stream;
    const size_t rd = static_cast<size_t>(rows) * d, cap = static_cast<size_t>(round_up(rows, 8)) * d;
    DevBuf<float> dx, dg, db;
    DevBuf<__half> dy;
    layernorm_f32_to_f16_run(to_device(dx, x, rd, s), to_device(dg, g, d, s), to_device(db, b, d, s), to_device(dy, y, cap, s),
                             rows, d, s, pdl != 0);
    WISB_CUDA(cudaMemcpyAsync(y, dy.p, cap * sizeof(__half), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_enc_layer(wisb_handle* h, int layer, int B, const float* x_in, float* x_out, void* stages_out, int32_t* plan_out) {
  return guarded(h, [&] {
    WISB_REQUIRE(h->blob != nullptr && x_in && x_out, "debug_enc_layer: bad arguments");
    WISB_REQUIRE(layer >= 0 && layer < h->dims.n_enc_layers, "debug_enc_layer: layer out of range");
    WISB_REQUIRE(B >= 1 && B <= 4096, "debug_enc_layer: B out of range");
    const int d = h->dims.d_model;
    const size_t md = static_cast<size_t>(B) * T_ENC_PAD * d;
    cudaStream_t s = h->stream;
    ensure_encoder(h, B);
    h->enc_valid = false;  // x now holds no features' rows
    h->mel_cache_B = 0;
    WISB_CUDA(cudaMemcpyAsync(h->x.p, x_in, md * sizeof(float), cudaMemcpyHostToDevice, s));
    // snapshots at byte offsets (units of md): xn1 0, qkv 2, vt 8, ctx 10, x after o-proj 12, xn2 16, fc1 output 18
    uint8_t* o = static_cast<uint8_t*>(stages_out);
    auto save = [&](size_t at, const void* src, size_t bytes) {
      WISB_CUDA(cudaMemcpyAsync(o + at * md, src, bytes, cudaMemcpyDeviceToHost, s));
    };
    const std::function<void(int)> snap = [&](int k) {
      switch (k) {
        case 0: save(0, h->xn.p, md * 2); break;
        case 1: save(2, h->qkv.p, md * 6); save(8, h->vt.p, md * 2); break;
        case 2: save(10, h->ctx.p, md * 2); break;
        case 3: save(12, h->x.p, md * 4); break;
        case 4: save(16, h->xn.p, md * 2); break;
        case 5: save(18, h->hbuf.p, md * 8); break;
        default: break;
      }
    };
    enc_layer_run(h, layer, B * T_ENC_PAD, o ? &snap : nullptr);
    WISB_CUDA(cudaMemcpyAsync(x_out, h->x.p, md * sizeof(float), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
    if (plan_out) {
      const EncLayerPlans& pl = h->enc_plans[layer];
      const GemmPlan* ps[4] = {&pl.qkv, &pl.o, &pl.fc1, &pl.fc2};
      for (int i = 0; i < 4; ++i) {
        plan_out[4 * i] = ps[i]->BN;
        plan_out[4 * i + 1] = ps[i]->mcast;
        plan_out[4 * i + 2] = ps[i]->k_splits;
        plan_out[4 * i + 3] = ps[i]->grid;
      }
    }
  });
}

int wisb_debug_forced_logits(wisb_handle* h, const float* mel, const int32_t* tokens, int n_tokens, float* logits_out) {
  return guarded(h, [&] {
    const Dims& dm = h->dims;
    WISB_REQUIRE(h->blob != nullptr && tokens != nullptr && logits_out != nullptr && n_tokens >= 1 && n_tokens <= dm.n_text_ctx, "bad arguments");
    cudaStream_t s = h->stream;
    const bool batched = h->decoder_batch == 2;
    encode_stage(h, upload_mel(h, mel, 1), false, 1, 0, 1, ckv_layout(h, !batched));
    DecodeCfg c;
    c.u0 = 0; c.n_utt = 1; c.B_total = 1; c.beam = 1; c.prompt_len = n_tokens; c.max_new = 1; c.max_hyp = 1; c.lp = 1.f;
    if (batched) {  // the batched pass, one row: position p of the token list per pass
      ensure_batch(h, MAX_BEAM, n_tokens);
      bind_batch_cross_kv(h, 0, 1);
      upload_prompts(h, tokens, nullptr, c);
      // `debug_chunk` positions per pass (1..8): > 1 feeds consecutive positions as rows of one pass, the way the prompt
      // prefix is prefilled (exercises the multi-row paths of the attention kernels under teacher forcing)
      const int chunk_max = std::max(1, std::min(h->debug_chunk, MAX_BEAM));
      batch_prefill(h, c, n_tokens, n_tokens, chunk_max, 1, true, nullptr, [&](int p, int chunk) {
        WISB_CUDA(cudaMemcpy2DAsync(logits_out + static_cast<size_t>(p) * dm.n_vocab, sizeof(float) * dm.n_vocab, h->blogits.p,
                                    sizeof(float) * dm.n_vocab_pad, sizeof(float) * dm.n_vocab, chunk, cudaMemcpyDeviceToHost, s));
      });
      WISB_CUDA(cudaStreamSynchronize(s));
      return;
    }
    persistent_setup(h, c, tokens, nullptr);
    for (int p = 0; p < n_tokens; ++p) {
      enqueue_decoder_forward(h, c, true);
      WISB_CUDA(cudaMemcpyAsync(logits_out + static_cast<size_t>(p) * dm.n_vocab, h->logits.p, sizeof(float) * dm.n_vocab, cudaMemcpyDeviceToHost, s));
      if (p + 1 < n_tokens) prefill_advance_run(h->tokens.p, h->prompt_dev.p, n_tokens, 1, 1, h->st.p, s);
    }
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_dec_pass(wisb_handle* h, const int32_t* prm, int n_prm, const int32_t* tokens, const int32_t* indir0,
                        const int32_t* indir1, const uint16_t* enc16, uint16_t* ckv_out, uint16_t* kcache, uint16_t* vcache,
                        float* x, float* logits) {
  return guarded(h, [&] {
    WISB_REQUIRE(h->blob != nullptr && prm != nullptr && n_prm == 7 && tokens && enc16 && ckv_out && kcache && vcache && x && logits,
                 "debug_dec_pass: bad arguments");
    const Dims& dm = h->dims;
    const int impl = prm[0], n_utt = prm[1], beam = prm[2], pf_len = prm[3], pos = prm[4], flip = prm[5], with_logits = prm[6];
    WISB_REQUIRE(impl == 0 || impl == 1, "debug_dec_pass: impl is 0 (SIMT) or 1 (warp-MMA)");
    WISB_REQUIRE(impl == 0 || h->mega_img.p != nullptr, "debug_dec_pass: the warp-MMA pass needs d_model <= 1280");
    WISB_REQUIRE(n_utt >= 1 && beam >= 1 && n_utt * beam <= DEC_MAX_ROWS, "debug_dec_pass: n_utt x beam must be 1..8");
    WISB_REQUIRE(pf_len >= 0 && pf_len <= MAX_BEAM && n_utt * pf_len <= DEC_MAX_ROWS, "debug_dec_pass: n_utt x pf_len must be <= 8");
    WISB_REQUIRE((flip == 0 || flip == 1) && (with_logits == 0 || with_logits == 1), "debug_dec_pass: flip and with_logits are 0 / 1");
    const int R = pf_len > 0 ? n_utt * pf_len : n_utt * beam;
    WISB_REQUIRE(pf_len > 0 || (pos >= 0 && pos < T_MAX), "debug_dec_pass: position outside 0..447");
    for (int r = 0; r < R; ++r)
      WISB_REQUIRE(tokens[r] >= 0 && tokens[r] < dm.n_vocab, "debug_dec_pass: token outside the vocabulary");
    if (pf_len == 0) {
      WISB_REQUIRE(indir0 != nullptr && indir1 != nullptr, "debug_dec_pass: a decoding step needs indir0 / indir1");
      for (int r = 0; r < R; ++r)
        for (int t = 0; t < pos; ++t)
          WISB_REQUIRE(indir0[r * T_MAX + t] >= 0 && indir0[r * T_MAX + t] < DEC_MAX_ROWS && indir1[r * T_MAX + t] >= 0 &&
                           indir1[r * T_MAX + t] < DEC_MAX_ROWS,
                       "debug_dec_pass: indirection entry outside the 8 cache slots");
    }
    cudaStream_t s = h->stream;
    const int d = dm.d_model, L = dm.n_dec_layers;
    // encoder rows -> enc_out -> cross K/V: first in the plain layout (returned), then in the layout the pass reads
    ensure_encoder(h, n_utt);
    h->enc_valid = false;  // these rows belong to no features: a later call must not reuse them
    h->mel_cache_B = 0;
    const size_t enc_elems = static_cast<size_t>(n_utt) * T_ENC_PAD * d;
    WISB_CUDA(cudaMemcpyAsync(h->enc_out.p, enc16, enc_elems * sizeof(__half), cudaMemcpyHostToDevice, s));
    const size_t ckv_elems = static_cast<size_t>(L) * 2 * enc_elems;
    h->plan_ckv.epi.kv_swizzle = 0;
    gemm_run(h->plan_ckv, s);
    WISB_CUDA(cudaMemcpyAsync(ckv_out, h->ckv.p, ckv_elems * sizeof(__half), cudaMemcpyDeviceToHost, s));
    const int saved_mma = h->mega_mma;
    h->mega_mma = impl;
    const int sw = ckv_layout(h, true);
    if (sw != 0) {
      h->plan_ckv.epi.kv_swizzle = sw;
      gemm_run(h->plan_ckv, s);
    }
    h->ckv_is_sw = sw;
    // the step's device state: position, indirection, tokens (prefill: the prompt rows), caches, sentinel outputs
    DecodeCfg c;
    c.u0 = 0; c.n_utt = n_utt; c.B_total = n_utt; c.beam = beam; c.prompt_len = pf_len + 1; c.max_new = 1; c.max_hyp = 1; c.lp = 1.f;
    const DecState st{pf_len > 0 ? 0 : pos, 0, 0, 0, 0};
    WISB_CUDA(cudaMemcpyAsync(h->st.p, &st, sizeof(DecState), cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(h->flip.p, &flip, sizeof(int), cudaMemcpyHostToDevice, s));
    std::vector<int> prompt;
    if (pf_len > 0) {
      prompt.assign(static_cast<size_t>(n_utt) * c.prompt_len, 0);
      for (int r = 0; r < R; ++r) prompt[(r / pf_len) * c.prompt_len + r % pf_len] = tokens[r];
      WISB_CUDA(cudaMemcpyAsync(h->prompt_dev.p, prompt.data(), prompt.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    } else {
      WISB_CUDA(cudaMemcpyAsync(h->tokens.p, tokens, R * sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(h->ind0.p, indir0, static_cast<size_t>(R) * T_MAX * sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(h->ind1.p, indir1, static_cast<size_t>(R) * T_MAX * sizeof(int), cudaMemcpyHostToDevice, s));
    }
    const size_t cache = static_cast<size_t>(L) * DEC_MAX_ROWS * T_MAX * d;
    const size_t xs = static_cast<size_t>(DEC_MAX_ROWS) * d, ls = static_cast<size_t>(DEC_MAX_ROWS) * dm.n_vocab_pad;
    WISB_CUDA(cudaMemcpyAsync(h->kcache.p, kcache, cache * sizeof(__half), cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(h->vcache.p, vcache, cache * sizeof(__half), cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(h->dx.p, x, xs * sizeof(float), cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(h->logits.p, logits, ls * sizeof(float), cudaMemcpyHostToDevice, s));
    try {
      upload_mega_layers(h, c);
      enqueue_decoder_forward(h, c, with_logits != 0, pf_len);
    } catch (...) {
      h->mega_mma = saved_mma;
      throw;
    }
    h->mega_mma = saved_mma;
    WISB_CUDA(cudaMemcpyAsync(kcache, h->kcache.p, cache * sizeof(__half), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(vcache, h->vcache.p, cache * sizeof(__half), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(x, h->dx.p, xs * sizeof(float), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(logits, h->logits.p, ls * sizeof(float), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

int wisb_debug_dec_batch_pass(wisb_handle* h, const int32_t* prm, int n_prm, const int32_t* tokens, const int32_t* row_pos,
                              const int32_t* indir0, const int32_t* indir1, const int32_t* done, const uint16_t* ckv,
                              uint16_t* kcache, uint16_t* vcache, float* x, float* logits, int64_t* geom_out, int32_t* plan_out) {
  return guarded(h, [&] {
    WISB_REQUIRE(h->blob != nullptr && prm != nullptr && n_prm == 16 && geom_out != nullptr, "debug_dec_batch_pass: bad arguments");
    const Dims& dm = h->dims;
    const int d = dm.d_model, L = dm.n_dec_layers;
    const int kind = prm[0], n_utt = prm[1], rpu = prm[2], slot_stride = prm[3], prompt_len = prm[4], p0 = prm[5],
              batch_rows = prm[6], t_need = prm[7], chunk_max = prm[8], flip = prm[9], with_logits = prm[10],
              cross_tc = prm[11], ckv_sw = prm[12], poison = prm[13], poison_slot = prm[14], poison_pos = prm[15];
    WISB_REQUIRE(kind >= 0 && kind <= 3, "debug_dec_batch_pass: kind 0 (step), 1 (prefill), 2 / 3 (wide prefill, batched / "
                                         "persistent cache)");
    WISB_REQUIRE(n_utt >= 1 && n_utt <= BD_CROSS_MAX_UTT,
                 "debug_dec_batch_pass: 1.." + std::to_string(BD_CROSS_MAX_UTT) + " windows in one pass");
    const bool wide = kind >= 2;
    WISB_REQUIRE(rpu >= 1 && rpu <= (wide ? T_MAX : MAX_BEAM), "debug_dec_batch_pass: 1..8 rows per window, 1..448 in a wide pass");
    const int R = n_utt * rpu;
    WISB_REQUIRE((flip == 0 || flip == 1) && (cross_tc == 0 || cross_tc == 1) && (ckv_sw == 0 || ckv_sw == 1) &&
                     (poison == 0 || poison == 1),
                 "debug_dec_batch_pass: flip, cross_tc, ckv_sw and poison are 0 / 1");
    WISB_REQUIRE(kind == 0 ? with_logits == 1 : kind == 1 ? (with_logits == 0 || with_logits == 1) : with_logits == 0,
                 "debug_dec_batch_pass: a step has logits, a wide pass none, a prefill pass 0 / 1");
    WISB_REQUIRE(ckv_sw == 0 || kind == 3, "debug_dec_batch_pass: only the persistent pass's cache pairs with swizzled cross K/V");
    WISB_REQUIRE(kind == 3 || (batch_rows >= 1 && batch_rows <= 4096 && t_need >= 1 && t_need <= T_MAX),
                 "debug_dec_batch_pass: batch_rows 1..4096, t_need 1..448");
    WISB_REQUIRE(kind != 0 || batch_rows >= R, "debug_dec_batch_pass: a step has more rows than batch_rows");
    WISB_REQUIRE(!wide || (chunk_max >= rpu && chunk_max <= T_MAX && static_cast<long long>(n_utt) * chunk_max <= 65536),
                 "debug_dec_batch_pass: a wide pass needs rows_per_utt <= chunk_max <= 448, n_utt x chunk_max <= 65536");
    WISB_REQUIRE(kind == 0 || (slot_stride >= 1 && prompt_len >= 1 && prompt_len <= T_MAX && p0 >= 0 && p0 + rpu <= prompt_len &&
                               p0 + rpu <= dm.n_text_ctx),
                 "debug_dec_batch_pass: prefill positions p0 .. p0 + rows_per_utt - 1 outside the prompt or n_text_ctx");
    // the geometry the pass will have: the workspaces' growth rules, applied before anything is allocated
    const int slots = kind == 3 ? DEC_MAX_ROWS : batch_rows_cap(h, batch_rows);
    const int t_cap = kind == 3 ? T_MAX : batch_tcap(h, t_need);
    const size_t layer_cache = static_cast<size_t>(slots) * t_cap * d;
    const int cap = wide ? prefill_rows_cap(h, n_utt * chunk_max) : slots;
    geom_out[0] = slots;
    geom_out[1] = t_cap;
    geom_out[2] = static_cast<int64_t>(layer_cache);
    geom_out[3] = cap;
    if (kcache == nullptr) return;  // geometry only: nothing allocated or launched
    WISB_REQUIRE(tokens && ckv && vcache && x && (with_logits == 0 || logits), "debug_dec_batch_pass: NULL argument");
    WISB_REQUIRE(R <= cap, "debug_dec_batch_pass: more rows than the workspaces hold");
    // every index the pass forms, against those sizes: positions < t_cap and < n_text_ctx, slots < the cache's
    const int n_pos = std::min(t_cap, dm.n_text_ctx);
    std::vector<char> wr(static_cast<size_t>(slots) * t_cap, 0);  // cells the pass writes
    if (kind == 0) {
      WISB_REQUIRE(row_pos && indir0 && indir1, "debug_dec_batch_pass: a step needs row_pos, indir0 and indir1");
      for (int r = 0; r < R; ++r) {
        WISB_REQUIRE(tokens[r] >= 0 && tokens[r] < dm.n_vocab && row_pos[r] >= 0 && row_pos[r] < n_pos,
                     "debug_dec_batch_pass: token / position out of range");
        for (int t = 0; t < row_pos[r]; ++t) {
          const size_t i = static_cast<size_t>(r) * T_MAX + t;
          WISB_REQUIRE(indir0[i] >= 0 && indir0[i] < slots && indir1[i] >= 0 && indir1[i] < slots,
                       "debug_dec_batch_pass: indirection entry outside the cache slots");
        }
        wr[static_cast<size_t>(r) * t_cap + row_pos[r]] = 1;
      }
    } else {
      WISB_REQUIRE(p0 + rpu <= n_pos, "debug_dec_batch_pass: prefill position outside the cache (t_cap) or n_text_ctx");
      WISB_REQUIRE(static_cast<long long>(n_utt - 1) * slot_stride < slots, "debug_dec_batch_pass: window slot outside the cache");
      for (int u = 0; u < n_utt; ++u)
        for (int p = p0; p < p0 + rpu; ++p) {
          const int tk = tokens[static_cast<size_t>(u) * prompt_len + p];
          WISB_REQUIRE(tk >= 0 && tk < dm.n_vocab, "debug_dec_batch_pass: token out of range");
          wr[static_cast<size_t>(u) * slot_stride * t_cap + p] = 1;
        }
    }
    if (poison)
      WISB_REQUIRE(poison_slot >= 0 && poison_slot < slots && poison_pos >= 0 && poison_pos < n_pos &&
                       !wr[static_cast<size_t>(poison_slot) * t_cap + poison_pos],
                   "debug_dec_batch_pass: the poison cell must be a cache cell the pass does not write");
    cudaStream_t s = h->stream;
    // workspaces and plans as the production callers make them (decode_batch / align_group / wide_prefill_run)
    ensure_search(h, n_utt);
    if (kind <= 2) ensure_batch(h, batch_rows, t_need);
    __half* kc = kind == 3 ? h->kcache.p : h->bkc.p;
    __half* vc = kind == 3 ? h->vcache.p : h->bvc.p;
    if (wide) ensure_prefill(h, n_utt * chunk_max, kc, vc, layer_cache, t_cap);
    WISB_REQUIRE((kind == 3 || (h->bd_rows == slots && h->bd_tcap == t_cap)) && (wide ? h->pf_rows : h->bd_rows) == cap,
                 "debug_dec_batch_pass: workspaces differ from the geometry reported");
    std::vector<BatchLayer>& layers = wide ? h->pf_layers : h->bd_layers;
    if (plan_out) {
      const GemmPlan* ps[7] = {&layers[0].qkv, &layers[0].o, &layers[0].cq, &layers[0].co, &layers[0].fc1, &layers[0].fc2,
                               &h->bd_vocab};
      for (int i = 0; i < 7; ++i) {
        const bool v = i < 6 || !wide;
        plan_out[4 * i] = v ? ps[i]->BN : 0;
        plan_out[4 * i + 1] = v ? ps[i]->mcast : 0;
        plan_out[4 * i + 2] = v ? ps[i]->k_splits : 0;
        plan_out[4 * i + 3] = v ? ps[i]->grid : 0;
      }
    }
    // caller state: cross K/V (the layout the pass reads), caches, row tables / search state
    ensure_encoder(h, n_utt);
    h->enc_valid = false;  // the cross K/V below belong to no features: a later call must not reuse them
    h->mel_cache_B = 0;
    const size_t ckv_elems = static_cast<size_t>(L) * 2 * n_utt * T_ENC_PAD * d;
    WISB_CUDA(cudaMemcpyAsync(h->ckv.p, ckv, ckv_elems * sizeof(__half), cudaMemcpyHostToDevice, s));
    h->ckv_is_sw = ckv_sw;
    const size_t cache = static_cast<size_t>(L) * layer_cache;
    WISB_CUDA(cudaMemcpyAsync(kc, kcache, cache * sizeof(__half), cudaMemcpyHostToDevice, s));
    WISB_CUDA(cudaMemcpyAsync(vc, vcache, cache * sizeof(__half), cudaMemcpyHostToDevice, s));
    int* tab_tok = wide ? h->ptok.p : h->tokens.p;
    int* tab_pos = wide ? h->ppos.p : h->row_pos.p;
    int* tab_slot = wide ? h->pslot.p : h->row_slot.p;
    if (poison && cap > R) {  // row-table entries >= R: one valid cell the pass does not write
      std::vector<int> t0(cap - R, 0), tp(cap - R, poison_pos), ts(cap - R, poison_slot);
      WISB_CUDA(cudaMemcpyAsync(tab_tok + R, t0.data(), t0.size() * sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(tab_pos + R, tp.data(), tp.size() * sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(tab_slot + R, ts.data(), ts.size() * sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaStreamSynchronize(s));  // (host temporaries)
    }
    DecodeCfg c{};
    c.u0 = 0; c.n_utt = n_utt; c.B_total = n_utt; c.max_new = 1; c.max_hyp = 1; c.lp = 1.f;
    c.beam = kind == 0 ? rpu : slot_stride;
    c.prompt_len = kind == 0 ? 1 : prompt_len;
    if (kind == 0) {
      WISB_CUDA(cudaMemcpyAsync(h->tokens.p, tokens, R * sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(h->row_pos.p, row_pos, R * sizeof(int), cudaMemcpyHostToDevice, s));
      std::vector<int> slot(R), dn(n_utt, 0);
      for (int r = 0; r < R; ++r) slot[r] = r;
      if (done) std::copy(done, done + n_utt, dn.begin());
      WISB_CUDA(cudaMemcpyAsync(h->row_slot.p, slot.data(), R * sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(h->done.p, dn.data(), n_utt * sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(h->ind0.p, indir0, static_cast<size_t>(R) * T_MAX * sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(h->ind1.p, indir1, static_cast<size_t>(R) * T_MAX * sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaMemcpyAsync(h->flip.p, &flip, sizeof(int), cudaMemcpyHostToDevice, s));
      WISB_CUDA(cudaStreamSynchronize(s));  // (host temporaries)
    } else {
      WISB_CUDA(cudaMemcpyAsync(h->prompt_dev.p, tokens, static_cast<size_t>(n_utt) * prompt_len * sizeof(int),
                                cudaMemcpyHostToDevice, s));
      prefill_rows_run(tab_tok, tab_pos, tab_slot, h->prompt_dev.p, prompt_len, n_utt, p0, rpu, slot_stride, s);
    }
    // poison: rows >= R of every activation workspace and partial slab NaN (all-ones bytes) for this pass, restored after
    float* wx = wide ? h->px.p : h->bx.p;
    struct Region {
      void* p;
      size_t bytes;
    };
    const size_t rd = static_cast<size_t>(R) * d, cd = static_cast<size_t>(cap) * d;
    std::vector<Region> regions;
    if (poison) {
      auto rows_of = [&](void* base, size_t esz, size_t width) {
        regions.push_back({static_cast<uint8_t*>(base) + esz * width * R, esz * width * (cap - R)});
      };
      rows_of(wx, 4, d);
      rows_of(wide ? static_cast<void*>(h->pxn.p) : h->bxn.p, 2, d);
      rows_of(wide ? static_cast<void*>(h->pq.p) : h->bq.p, 4, d);
      rows_of(wide ? static_cast<void*>(h->pctx.p) : h->bctx.p, 2, d);
      rows_of(wide ? static_cast<void*>(h->ph.p) : h->bh.p, 2, 4 * static_cast<size_t>(d));
      float* part = wide ? h->ppart.p : h->bpart.p;
      for (int sl = 0; sl < 8; ++sl) regions.push_back({part + sl * cd + rd, 4 * (cd - rd)});
    }
    size_t saved_bytes = 0;
    for (const Region& g : regions) saved_bytes += g.bytes;
    DevBuf<uint8_t> saved;
    saved.ensure(saved_bytes);
    {
      size_t at = 0;
      for (const Region& g : regions) {
        WISB_CUDA(cudaMemcpyAsync(saved.p + at, g.p, g.bytes, cudaMemcpyDeviceToDevice, s));
        WISB_CUDA(cudaMemsetAsync(g.p, 0xFF, g.bytes, s));
        at += g.bytes;
      }
    }
    // the pass, through the argument builders of its production caller
    const int saved_tc = h->cross_tc;
    h->cross_tc = cross_tc;
    try {
      BatchArgs a;
      if (kind == 0) {
        bind_batch_cross_kv(h, 0, n_utt);
        a = batch_step_args(h, c);
      } else if (kind == 1) {
        bind_batch_cross_kv(h, 0, n_utt);
        a = batch_prefill_args(h, c, rpu, with_logits != 0);
      } else {
        for (int i = 0; i < L; ++i) bind_cross_kv(h, h->pf_layers[i], i, c.u0, c.B_total);
        a = wide_prefill_args(h, c, rpu, t_cap);
      }
      batch_pass_run(a, layers.data(), L, s);
    } catch (...) {
      h->cross_tc = saved_tc;
      throw;
    }
    h->cross_tc = saved_tc;
    {
      size_t at = 0;
      for (const Region& g : regions) {
        WISB_CUDA(cudaMemcpyAsync(g.p, saved.p + at, g.bytes, cudaMemcpyDeviceToDevice, s));
        at += g.bytes;
      }
    }
    WISB_CUDA(cudaMemcpyAsync(kcache, kc, cache * sizeof(__half), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(vcache, vc, cache * sizeof(__half), cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaMemcpyAsync(x, wx, rd * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (with_logits)  // (columns >= n_vocab of the caller's rows stay as they were)
      WISB_CUDA(cudaMemcpy2DAsync(logits, sizeof(float) * dm.n_vocab_pad, h->blogits.p, sizeof(float) * dm.n_vocab_pad,
                                  sizeof(float) * dm.n_vocab, R, cudaMemcpyDeviceToHost, s));
    WISB_CUDA(cudaStreamSynchronize(s));
  });
}

}  // extern "C"
