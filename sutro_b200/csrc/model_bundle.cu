// sutro_b200 — a model on disk and the strings-only call: what a host WITHOUT Python binds.
//
// The reference's client sends {model, inputs, system_prompt, json_schema, sampling_params}
// and the service does the rest (sutro/sdk.py:196-223).  Behind the C-ABI that "rest" is:
//   sb200_model_open    a bundle directory (manifest.json + data.bin written by
//                       sutro_b200/bundle.py: architecture, weights in engine layout, RoPE
//                       tables, tokenizer tables, special-token ids, template family)
//                       -> weights in HBM, engine + GPU tokenizer created
//   sb200_model_infer   system prompt + JSON schema text + rows (Arrow-style bytes/offsets)
//                       -> chat template rendered and tokenised, schema compiled
//                       (schema_compile.cu), jump-forward plan derived from the automaton,
//                       sb200_infer_text run, results returned as host buffers
// Everything numerical still happens in the kernels; this file is host plumbing that the
// Python host (engine.py: _template_tokens / _jump_plan / _job_options) does the same way —
// tests/test_c_host_gpu.py runs a C program through this path and compares its outputs with
// LocalEngine.generate on the same rows.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/sutro_b200.h"
#include "common.cuh"
#include "dev_buf.h"
#include "json_mini.h"
#include "kernels.h"

namespace sb {
namespace {

using json::JVal;

struct Tensor {
  int64_t offset = 0, bytes = 0;
};

struct Model {
  int device = 0;
  std::string family;
  sb200_engine_config cfg{};
  std::map<std::string, int> specials;
  void* engine = nullptr;
  void* tokenizer = nullptr;
  std::vector<void*> dev_allocs;
  std::vector<const void*> ln1, ln2, wqkv, wo, wgu, wd, qn, kn;
  ~Model() {
    if (engine) sb200_engine_destroy(engine);
    if (tokenizer) sb200_tokenizer_destroy(tokenizer);
    for (void* p : dev_allocs) cudaFree(p);
  }
};

int read_file(const std::string& path, std::vector<char>* out) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) {
    set_last_error("model_open: cannot open %s", path.c_str());
    return -1;
  }
  fseek(f, 0, SEEK_END);
  const long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  out->resize(n > 0 ? n : 0);
  const size_t got = n > 0 ? fread(out->data(), 1, n, f) : 0;
  fclose(f);
  if (static_cast<long>(got) != n) {
    set_last_error("model_open: short read on %s", path.c_str());
    return -1;
  }
  return 0;
}

long long num(const JVal& o, const char* k) {
  const JVal* v = o.get(k);
  if (!v || v->t != JVal::Num) json::fail(std::string("manifest: missing number '") + k + "'");
  return static_cast<long long>(strtod(v->s.c_str(), nullptr));
}
double fnum(const JVal& o, const char* k) {
  const JVal* v = o.get(k);
  if (!v || v->t != JVal::Num) json::fail(std::string("manifest: missing number '") + k + "'");
  return strtod(v->s.c_str(), nullptr);
}

// ---- tokenise host strings with the GPU tokenizer (template pieces, forced schema text) ----
int encode_texts(Model* m, const std::vector<std::string>& texts,
                 std::vector<std::vector<int32_t>>* out) {
  out->assign(texts.size(), {});
  if (texts.empty()) return 0;
  std::vector<int64_t> off(texts.size() + 1, 0);
  std::string blob;
  for (size_t i = 0; i < texts.size(); ++i) {
    blob += texts[i];
    off[i + 1] = static_cast<int64_t>(blob.size());
  }
  const int64_t nb = static_cast<int64_t>(blob.size());
  cudaStream_t stream = static_cast<cudaStream_t>(sb200_engine_stream(m->engine));
  const size_t n1 = texts.size() + 1;
  DevBuf d_text, d_off, d_toff, d_tok;
  if (d_text.alloc(nb) || d_off.alloc(n1 * 8) || d_toff.alloc(n1 * 8) || d_tok.alloc(nb * 4)) {
    set_last_error("model: out of device memory while tokenising template text");
    return -1;
  }
  auto cuda_error = [] {
    set_last_error("model: CUDA error while tokenising template text");
    return -1;
  };
  const cudaMemcpyKind h2d = cudaMemcpyHostToDevice, d2h = cudaMemcpyDeviceToHost;
  if ((nb && cudaMemcpyAsync(d_text.p, blob.data(), nb, h2d, stream) != cudaSuccess) ||
      cudaMemcpyAsync(d_off.p, off.data(), n1 * 8, h2d, stream) != cudaSuccess)
    return cuda_error();
  if (sb200_tokenizer_encode(m->tokenizer, d_text.as<uint8_t>(), nb, d_off.as<int64_t>(),
                             static_cast<int64_t>(texts.size()), d_tok.as<int32_t>(),
                             d_toff.as<int64_t>(), stream))
    return -1;
  std::vector<int64_t> toff(n1);
  if (cudaMemcpyAsync(toff.data(), d_toff.p, n1 * 8, d2h, stream) != cudaSuccess ||
      cudaStreamSynchronize(stream) != cudaSuccess)
    return cuda_error();
  std::vector<int32_t> toks(toff.back() > 0 ? toff.back() : 0);
  if (!toks.empty() &&
      (cudaMemcpyAsync(toks.data(), d_tok.p, toks.size() * 4, d2h, stream) != cudaSuccess ||
       cudaStreamSynchronize(stream) != cudaSuccess))
    return cuda_error();
  for (size_t i = 0; i < texts.size(); ++i)
    (*out)[i].assign(toks.begin() + toff[i], toks.begin() + toff[i + 1]);
  return 0;
}

// template pieces -> token ids: a piece naming a special token maps to its id, anything else
// is tokenised on its own (sutro_b200/vocab.py chat_template / GpuTokenizer.encode_pieces)
int encode_pieces(Model* m, const std::vector<std::string>& pieces, std::vector<int32_t>* out) {
  std::vector<std::string> texts;
  for (auto& p : pieces)
    if (!m->specials.count(p)) texts.push_back(p);
  std::vector<std::vector<int32_t>> enc;
  if (encode_texts(m, texts, &enc)) return -1;
  out->clear();
  size_t k = 0;
  for (auto& p : pieces) {
    auto it = m->specials.find(p);
    if (it != m->specials.end()) out->push_back(it->second);
    else {
      out->insert(out->end(), enc[k].begin(), enc[k].end());
      ++k;
    }
  }
  return 0;
}

void chat_template(const Model& m, const char* system_prompt, std::vector<std::string>* pre,
                   std::vector<std::string>* suf) {
  const bool sys = system_prompt && system_prompt[0];
  pre->clear();
  suf->clear();
  if (m.cfg.embedding_model) {
    *suf = {m.family == "qwen3" ? "<|endoftext|>" : "<|end_of_text|>"};
    return;
  }
  if (m.family == "qwen3") {  // ChatML
    if (sys) *pre = {"<|im_start|>", std::string("system\n") + system_prompt, "<|im_end|>", "\n"};
    pre->push_back("<|im_start|>");
    pre->push_back("user\n");
    *suf = {"<|im_end|>", "\n", "<|im_start|>", "assistant\n"};
    return;
  }
  *pre = {"<|begin_of_text|>"};  // Llama-3 headers
  if (sys) {
    for (const char* p : {"<|start_header_id|>", "system", "<|end_header_id|>"}) pre->push_back(p);
    pre->push_back(std::string("\n\n") + system_prompt);
    pre->push_back("<|eot_id|>");
  }
  for (const char* p : {"<|start_header_id|>", "user", "<|end_header_id|>", "\n\n"}) pre->push_back(p);
  *suf = {"<|eot_id|>", "<|start_header_id|>", "assistant", "<|end_header_id|>", "\n\n"};
}

bool valid_utf8(const std::string& s) {
  size_t i = 0;
  while (i < s.size()) {
    const unsigned char c = s[i];
    int n = c < 0x80 ? 0 : (c >> 5) == 6 ? 1 : (c >> 4) == 14 ? 2 : (c >> 3) == 30 ? 3 : -1;
    if (n < 0 || i + n >= s.size() + (n == 0 ? 1 : 0)) return false;
    for (int k = 1; k <= n; ++k)
      if ((static_cast<unsigned char>(s[i + k]) & 0xC0) != 0x80) return false;
    i += n + 1;
  }
  return true;
}

// ByteDFA.forced_run: follow a state while exactly one byte keeps the automaton alive and the
// state is not accepting
void forced_run(const int32_t* trans, const uint8_t* accept, int state, std::string* run, int* end) {
  run->clear();
  int s = state;
  while (!accept[s]) {
    int cnt = 0, byte = -1;
    const int32_t* row = trans + static_cast<size_t>(s) * 256;
    for (int b = 0; b < 256 && cnt < 2; ++b)
      if (row[b] >= 0) {
        ++cnt;
        byte = b;
      }
    if (cnt != 1) break;
    run->push_back(static_cast<char>(byte));
    s = row[byte];
  }
  *end = s;
}

}  // namespace
}  // namespace sb

using namespace sb;

extern "C" {

int sb200_model_open(const char* dir, int device, int max_slots, int max_prefill_tokens,
                     int64_t kv_pages, void** out) {
  if (out) *out = nullptr;
  if (!dir || !out) {
    set_last_error("model_open: null argument");
    return -1;
  }
  std::vector<char> man, data;
  if (read_file(std::string(dir) + "/manifest.json", &man)) return -1;
  auto m = std::unique_ptr<Model>(new Model());
  m->device = device;
  try {
    const JVal root = json::parse(man.data(), man.size());
    if (num(root, "format") != 1) json::fail("manifest: unknown format version");
    const JVal* spec = root.get("spec");
    const JVal* tens = root.get("tensors");
    const JVal* spc = root.get("specials");
    if (!spec || !tens || !spc) json::fail("manifest: spec / tensors / specials missing");
    const JVal* fam = spec->get("family");
    m->family = fam && fam->t == JVal::Str ? fam->s : "qwen3";
    sb200_engine_config& c = m->cfg;
    c.n_layers = static_cast<int>(num(*spec, "n_layers"));
    c.d_model = static_cast<int>(num(*spec, "d_model"));
    c.n_q_heads = static_cast<int>(num(*spec, "n_q_heads"));
    c.n_kv_heads = static_cast<int>(num(*spec, "n_kv_heads"));
    c.d_ff = static_cast<int>(num(*spec, "d_ff"));
    c.vocab = static_cast<int>(num(*spec, "vocab_size"));
    c.max_position = static_cast<int>(num(*spec, "max_position"));
    c.rms_eps = static_cast<float>(fnum(*spec, "rms_eps"));
    c.qk_norm = static_cast<int>(num(*spec, "qk_norm"));
    c.embedding_model = static_cast<int>(num(*spec, "embedding_model"));
    c.eos_id = static_cast<int>(num(*spec, "eos_id"));
    c.max_slots = max_slots > 0 ? max_slots : 512;
    // the default step holds one row of up to 32,768 tokens; longer rows are prefilled in chunks
    c.max_prefill_tokens = max_prefill_tokens > 0
                               ? max_prefill_tokens
                               : std::max(8192, std::min(c.max_position, 32768));
    c.logit_chunk_rows = 1024;
    c.min_admit_rows = std::max(1, c.max_slots / 4);
    for (auto& kv : spc->o) m->specials[kv.first] = static_cast<int>(strtod(kv.second.s.c_str(), nullptr));

    if (read_file(std::string(dir) + "/data.bin", &data)) return -1;
    SB_CUDA_CHECK(cudaSetDevice(device));
    auto region = [&](const std::string& name, const char** host, int64_t* bytes) {
      const JVal* t = tens->get(name);
      if (!t) json::fail("manifest: tensor '" + name + "' missing");
      const int64_t off = num(*t, "offset"), nb = num(*t, "bytes");
      if (off < 0 || nb < 0 || off + nb > static_cast<int64_t>(data.size()))
        json::fail("manifest: tensor '" + name + "' outside data.bin");
      *host = data.data() + off;
      *bytes = nb;
    };
    auto to_dev = [&](const std::string& name) -> const void* {
      const char* h;
      int64_t nb;
      region(name, &h, &nb);
      void* d = nullptr;
      if (cudaMalloc(&d, nb ? nb : 1) != cudaSuccess ||
          cudaMemcpy(d, h, nb, cudaMemcpyHostToDevice) != cudaSuccess)
        json::fail("out of device memory loading '" + name + "'");
      m->dev_allocs.push_back(d);
      return d;
    };
    sb200_engine_weights w{};
    w.embed = to_dev("embed");
    w.lm_head = tens->has("lm_head") ? to_dev("lm_head") : w.embed;
    w.final_norm = to_dev("final_norm");
    w.rope_cos = to_dev("rope_cos");
    w.rope_sin = to_dev("rope_sin");
    for (int l = 0; l < c.n_layers; ++l) {
      const std::string p = "layers." + std::to_string(l) + ".";
      m->ln1.push_back(to_dev(p + "ln1"));
      m->ln2.push_back(to_dev(p + "ln2"));
      m->wqkv.push_back(to_dev(p + "wqkv"));
      m->wo.push_back(to_dev(p + "wo"));
      m->wgu.push_back(to_dev(p + "wgu"));
      m->wd.push_back(to_dev(p + "wd"));
      if (c.qk_norm) {
        m->qn.push_back(to_dev(p + "q_norm"));
        m->kn.push_back(to_dev(p + "k_norm"));
      }
    }
    w.ln1 = m->ln1.data(), w.ln2 = m->ln2.data(), w.wqkv = m->wqkv.data(), w.wo = m->wo.data();
    w.wgu = m->wgu.data(), w.wd = m->wd.data();
    w.q_norm = c.qk_norm ? m->qn.data() : nullptr;
    w.k_norm = c.qk_norm ? m->kn.data() : nullptr;
    if (kv_pages <= 0) {  // 80 % of what is free after the weights, capped at every slot full
      size_t free_b = 0, total_b = 0;
      SB_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
      const int64_t page_bytes = 2LL * c.n_layers * kv_page_elems(c.n_kv_heads);  // all layers, bf16
      const int64_t t_max = std::max(c.max_prefill_tokens, c.max_slots);
      const int64_t act = t_max * 2LL * (2LL * c.d_model + (c.n_q_heads + 2LL * c.n_kv_heads) * kHeadDim +
                                         c.n_q_heads * kHeadDim + c.d_ff) +
                          std::min<int64_t>(1024, c.max_slots) * 4LL * c.vocab;
      kv_pages = static_cast<int64_t>((static_cast<double>(free_b) - act) * 0.8) / page_bytes;
      kv_pages = std::min<int64_t>(kv_pages, static_cast<int64_t>(c.max_slots) * (c.max_position / 16 + 1) + 64);
    }
    if (kv_pages < 8) json::fail("not enough device memory for a KV pool");
    c.num_pages = kv_pages;
    if (sb200_engine_create(&c, &w, &m->engine)) return -1;
    // tokenizer tables (host arrays)
    const char *merges, *cls, *tokb, *toko, *mids = nullptr;
    int64_t nb_merges, nb_cls, nb_tokb, nb_toko, nb_mids = 0;
    region("tok.merges", &merges, &nb_merges);
    region("tok.cls_table", &cls, &nb_cls);
    region("tok.bytes", &tokb, &nb_tokb);
    region("tok.offsets", &toko, &nb_toko);
    if (tens->has("tok.merged_ids")) region("tok.merged_ids", &mids, &nb_mids);
    const JVal* tk = root.get("tokenizer");
    const int digits = tk ? static_cast<int>(num(*tk, "digits")) : 1;
    if (nb_toko != (c.vocab + 1) * 4LL) json::fail("manifest: tok.offsets has the wrong size");
    if (sb200_tokenizer_create(reinterpret_cast<const int32_t*>(merges), static_cast<int>(nb_merges / 8),
                               reinterpret_cast<const int32_t*>(mids),
                               reinterpret_cast<const uint8_t*>(cls), digits,
                               reinterpret_cast<const uint8_t*>(tokb),
                               reinterpret_cast<const int32_t*>(toko), c.vocab, &m->tokenizer))
      return -1;
    if (tens->has("tok.override_ids")) {   // the tokenizer file sets ignore_merges
      const char *ot, *oo, *oi;
      int64_t nb_ot, nb_oo, nb_oi;
      region("tok.override_tokens", &ot, &nb_ot);
      region("tok.override_offsets", &oo, &nb_oo);
      region("tok.override_ids", &oi, &nb_oi);
      if (nb_oo != nb_oi + 4) json::fail("manifest: tok.override_offsets has the wrong size");
      if (sb200_tokenizer_set_word_overrides(m->tokenizer, reinterpret_cast<const int32_t*>(ot),
                                             reinterpret_cast<const int32_t*>(oo),
                                             reinterpret_cast<const int32_t*>(oi),
                                             static_cast<int>(nb_oi / 4)))
        return -1;
    }
    if (sb200_engine_set_vocab(m->engine, reinterpret_cast<const uint8_t*>(tokb),
                               reinterpret_cast<const int32_t*>(toko)))
      return -1;
  } catch (const json::SchemaFail& e) {
    set_last_error("model_open: %s", e.msg.c_str());
    return -1;
  }
  *out = m.release();
  return 0;
}

void sb200_model_close(void* model) { delete static_cast<Model*>(model); }
void* sb200_model_engine(void* model) { return model ? static_cast<Model*>(model)->engine : nullptr; }
void* sb200_model_tokenizer(void* model) {
  return model ? static_cast<Model*>(model)->tokenizer : nullptr;
}

int sb200_model_infer(void* model, const char* system_prompt_utf8, const char* json_schema_utf8,
                      int64_t schema_len, const sb200_fsm_limits* limits, int max_new_tokens,
                      const sb200_job* sampling, const uint8_t* rows_bytes,
                      const int64_t* rows_offsets, int64_t n_rows, int want_logprobs,
                      sb200_result** out, sb200_job_stats* stats) {
  if (out) *out = nullptr;
  if (!model || !out) {
    set_last_error("model_infer: null argument");
    return -1;
  }
  Model* m = static_cast<Model*>(model);
  SB_CUDA_CHECK(cudaSetDevice(m->device));
  // ---- prompt framing ----
  std::vector<std::string> pre_p, suf_p;
  chat_template(*m, system_prompt_utf8, &pre_p, &suf_p);
  std::vector<int32_t> pre, suf;
  if (encode_pieces(m, pre_p, &pre) || encode_pieces(m, suf_p, &suf)) return -1;
  // ---- output_schema -> automaton -> jump-forward plan ----
  void* schema = nullptr;
  struct SchemaGuard {
    void*& s;
    ~SchemaGuard() {
      if (s) sb200_schema_destroy(s);
    }
  } guard{schema};
  const int32_t* trans = nullptr;
  const uint8_t *accept = nullptr, *fin = nullptr;
  int n_states = 0, start = 0;
  const bool constrained = json_schema_utf8 && schema_len > 0 && !m->cfg.embedding_model;
  if (constrained) {
    const int rc = sb200_schema_compile(json_schema_utf8, schema_len, limits, &schema);
    if (rc) return rc;
    sb200_schema_tables(schema, &trans, &accept, &fin, &n_states, &start);
  }
  if (max_new_tokens <= 0) {  // the SDK's default budget (sdk.py _default_max_new_tokens)
    const int cap = std::max(16, std::min(m->cfg.max_position, 4096) / 2);
    const int64_t longest = constrained ? sb200_schema_longest_path(schema) : -1;
    max_new_tokens = longest >= 0 ? static_cast<int>(std::min<int64_t>(std::max<int64_t>(longest, 8), cap))
                                  : std::min(512, cap);
  }
  sb200_job job{};
  if (sampling) {
    job.temperature = sampling->temperature, job.top_k = sampling->top_k, job.top_p = sampling->top_p;
    job.seed = sampling->seed, job.seed_per_row = sampling->seed_per_row;
    job.ignore_eos = sampling->ignore_eos;
    job.progress = sampling->progress, job.progress_user = sampling->progress_user;
    job.profile = sampling->profile;
    job.presence_penalty = sampling->presence_penalty;
    job.frequency_penalty = sampling->frequency_penalty;
    job.repetition_penalty = sampling->repetition_penalty;
    job.min_p = sampling->min_p;
  }
  job.truncate_rows = sampling ? sampling->truncate_rows : 1;
  if (!sampling) job.truncate_rows = 1;
  job.share_prefix = 1;
  job.max_new_tokens = max_new_tokens;
  std::vector<int32_t> tail_off, tail_tok;
  if (constrained) {
    job.fsm_trans = trans, job.fsm_accept = accept, job.fsm_final = fin;
    job.fsm_states = n_states, job.fsm_start = start;
    // engine.py _jump_plan: the forced output prefix rides with the prompt, terminal tails are
    // appended by the sampler
    std::string prefix;
    int start_after = start;
    forced_run(trans, accept, start, &prefix, &start_after);
    std::vector<std::string> texts{prefix};
    std::vector<int> tail_state;
    for (int s = 0; s < n_states; ++s) {
      std::string run;
      int end;
      forced_run(trans, accept, s, &run, &end);
      if (!run.empty() && fin[end]) {
        texts.push_back(run);
        tail_state.push_back(s);
      }
    }
    bool fully_forced = fin[start_after] != 0;
    for (int s : tail_state) fully_forced = fully_forced || s == start_after;
    bool utf8_ok = true;
    for (auto& t : texts) utf8_ok = utf8_ok && valid_utf8(t);
    if (utf8_ok && !fully_forced && (!prefix.empty() || !tail_state.empty())) {
      std::vector<std::vector<int32_t>> enc;
      if (encode_texts(m, texts, &enc)) return -1;
      if (static_cast<int>(enc[0].size()) < max_new_tokens) {
        tail_off.assign(n_states + 1, 0);
        size_t k = 0;
        for (int s = 0; s < n_states; ++s) {
          if (k < tail_state.size() && tail_state[k] == s) {
            tail_tok.insert(tail_tok.end(), enc[k + 1].begin(), enc[k + 1].end());
            ++k;
          }
          tail_off[s + 1] = static_cast<int32_t>(tail_tok.size());
        }
        if (tail_tok.empty()) tail_tok.push_back(0);
        suf.insert(suf.end(), enc[0].begin(), enc[0].end());
        job.fsm_start = start_after;
        job.n_forced_prefix = static_cast<int>(enc[0].size());
        job.fsm_tail_off = tail_off.data();
        job.fsm_tail_tok = tail_tok.data();
      }
    }
  }
  job.prefix_tokens = pre.data(), job.n_prefix = static_cast<int>(pre.size());
  job.suffix_tokens = suf.data(), job.n_suffix = static_cast<int>(suf.size());
  return sb200_infer_text(m->engine, m->tokenizer, rows_bytes, rows_offsets, n_rows, &job, 1,
                          want_logprobs, out, stats);
}

}  // extern "C"
