// HF-layout checkpoint loading (SURVEY.md §8f-2 "next": real weights).  The reference mounts a model
// directory into the backend pod (internal/modelcontroller/model_source.go:231-287, hf:// / pvc:// sources)
// and vLLM reads its *.safetensors; the in-process engine reads the same files itself:
//   <dir>/config.json                       -> b200_config (b200_config_from_hf)
//   <dir>/model.safetensors[.index.json]    -> engine tensors (b200_engine_load_safetensors)
// q/k/v and gate/up projections are fused on load into the engine's wqkv / wgu layout (same row order as
// vLLM's merged qkv_proj / gate_up_proj, model_executor/models/llama.py:81-121,157-161).
#include <cuda_runtime.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <math.h>
#include <string.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/b200engine.h"
#include "errors.h"
#include "hostutil.h"

namespace b200 {
namespace {

struct StTensor {
  std::string dtype;
  std::vector<int64_t> shape;
  size_t begin = 0, end = 0;  // byte offsets inside the data section
};

struct StFile {
  int fd = -1;
  const uint8_t* map = nullptr;
  size_t size = 0, data_off = 0;
  std::map<std::string, StTensor> tensors;
  ~StFile() {
    if (map) munmap(const_cast<uint8_t*>(map), size);
    if (fd >= 0) close(fd);
  }
  bool open_file(const std::string& path, std::string* err) {
    fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) { *err = "cannot open " + path; return false; }
    struct stat st;
    if (fstat(fd, &st) || st.st_size < 8) { *err = "bad safetensors file " + path; return false; }
    size = static_cast<size_t>(st.st_size);
    void* p = mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
    if (p == MAP_FAILED) { *err = "mmap failed for " + path; return false; }
    map = static_cast<const uint8_t*>(p);
    uint64_t hlen = 0;
    memcpy(&hlen, map, 8);
    if (hlen > size - 8) { *err = "safetensors header length out of range in " + path; return false; }
    data_off = 8 + static_cast<size_t>(hlen);
    JVal root;
    std::string jerr;
    if (!JParser(reinterpret_cast<const char*>(map + 8), static_cast<size_t>(hlen)).parse(&root, &jerr) || root.type != JVal::Obj) {
      *err = "safetensors header of " + path + ": " + jerr;
      return false;
    }
    for (auto& kv : root.obj) {
      if (kv.first == "__metadata__") continue;
      StTensor t;
      const JVal* dt = kv.second.get("dtype");
      const JVal* sh = kv.second.get("shape");
      const JVal* off = kv.second.get("data_offsets");
      if (!dt || dt->type != JVal::Str || !sh || sh->type != JVal::Arr || !off || off->type != JVal::Arr || off->arr.size() != 2) {
        *err = "malformed entry " + kv.first + " in " + path;
        return false;
      }
      t.dtype = dt->str;
      // checkpoints are untrusted input: every number must be a non-negative integer below 2^53, offsets must lie inside
      // the data section (compared without forming data_off + end, which could wrap), shape products must not overflow
      auto as_index = [](const JVal& v, uint64_t* out) {
        if (v.type != JVal::Num || !(v.num >= 0.0) || v.num >= 9007199254740992.0 || v.num != floor(v.num)) return false;
        *out = static_cast<uint64_t>(v.num);
        return true;
      };
      uint64_t b = 0, e = 0, elems = 1;
      bool ok = as_index(off->arr[0], &b) && as_index(off->arr[1], &e);
      for (auto& d : sh->arr) {
        uint64_t dim = 0;
        if (!ok || !as_index(d, &dim) || (dim != 0 && elems > (1ull << 53) / dim)) { ok = false; break; }
        elems *= dim;
        t.shape.push_back(static_cast<int64_t>(dim));
      }
      const uint64_t data_len = static_cast<uint64_t>(size - data_off);
      if (!ok || e < b || e > data_len) { *err = "shape or data_offsets out of range for " + kv.first; return false; }
      t.begin = static_cast<size_t>(b);
      t.end = static_cast<size_t>(e);
      tensors[kv.first] = t;
    }
    return true;
  }
};

bool read_text(const std::string& path, std::string* out) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  char buf[65536];
  size_t n;
  out->clear();
  while ((n = fread(buf, 1, sizeof(buf), f)) > 0) out->append(buf, n);
  fclose(f);
  return true;
}

bool is_dir(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
}

size_t dtype_size(const std::string& d) { return d == "BF16" || d == "F16" ? 2 : d == "F32" ? 4 : 0; }

inline uint16_t f32_to_bf16(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40);  // NaN
  u += 0x7fffu + ((u >> 16) & 1u);
  return static_cast<uint16_t>(u >> 16);
}
inline float f16_to_f32(uint16_t h) {
  const uint32_t s = (h & 0x8000u) << 16, e = (h >> 10) & 0x1f, m = h & 0x3ffu;
  uint32_t u;
  if (e == 0) {
    if (m == 0) u = s;
    else {
      int sh = 0;
      uint32_t mm = m;
      while (!(mm & 0x400u)) { mm <<= 1; ++sh; }
      u = s | ((113 - sh) << 23) | ((mm & 0x3ffu) << 13);
    }
  } else if (e == 31) u = s | 0x7f800000u | (m << 13);
  else u = s | ((e + 112) << 23) | (m << 13);
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// All shards of a checkpoint: tensor name -> (file, entry)
struct Checkpoint {
  std::vector<std::unique_ptr<StFile>> files;
  std::map<std::string, std::pair<StFile*, const StTensor*>> index;
  bool open_path(const std::string& path, std::string* err) {
    std::vector<std::string> shard_paths;
    if (is_dir(path)) {
      std::string idx;
      if (read_text(path + "/model.safetensors.index.json", &idx)) {
        JVal root;
        std::string jerr;
        if (!JParser(idx.data(), idx.size()).parse(&root, &jerr)) { *err = "index json: " + jerr; return false; }
        const JVal* wm = root.get("weight_map");
        if (!wm || wm->type != JVal::Obj) { *err = "index json has no weight_map"; return false; }
        std::map<std::string, bool> seen;
        for (auto& kv : wm->obj)
          if (kv.second.type == JVal::Str && !seen[kv.second.str]) {
            seen[kv.second.str] = true;
            shard_paths.push_back(path + "/" + kv.second.str);
          }
      } else {
        shard_paths.push_back(path + "/model.safetensors");
      }
    } else {
      shard_paths.push_back(path);
    }
    for (auto& sp : shard_paths) {
      files.emplace_back(new StFile());
      if (!files.back()->open_file(sp, err)) return false;
      for (auto& kv : files.back()->tensors) index[kv.first] = {files.back().get(), &kv.second};
    }
    return true;
  }
};

// Copy a [rows, cols] checkpoint tensor into rows [row0, row0+rows) of a bf16 device matrix with `cols` columns.
int copy_rows(const Checkpoint& ck, const std::string& name, void* dev_base, size_t dev_bytes, int64_t row0, int64_t rows,
              int64_t cols, std::string* err) {
  auto it = ck.index.find(name);
  if (it == ck.index.end()) { *err = "missing tensor " + name; return B200_ERR_NOT_FOUND; }
  const StTensor& t = *it->second.second;
  const StFile& f = *it->second.first;
  int64_t n = 1;
  for (auto d : t.shape) n *= d;
  const int64_t trows = t.shape.size() == 2 ? t.shape[0] : 1, tcols = t.shape.size() == 2 ? t.shape[1] : n;
  if (trows != rows || tcols != cols) {
    *err = name + ": shape [" + std::to_string(trows) + "," + std::to_string(tcols) + "] != expected [" + std::to_string(rows) + "," + std::to_string(cols) + "]";
    return B200_ERR_INVALID;
  }
  const size_t es = dtype_size(t.dtype);
  if (!es || t.end - t.begin != static_cast<size_t>(n) * es) { *err = name + ": unsupported dtype " + t.dtype; return B200_ERR_INVALID; }
  const size_t dst_off = static_cast<size_t>(row0) * cols * 2;
  if (dst_off + static_cast<size_t>(n) * 2 > dev_bytes) { *err = name + ": does not fit the engine tensor"; return B200_ERR_INVALID; }
  const uint8_t* src = f.map + f.data_off + t.begin;
  uint8_t* dst = static_cast<uint8_t*>(dev_base) + dst_off;
  cudaError_t ce;
  if (t.dtype == "BF16") {
    ce = cudaMemcpy(dst, src, static_cast<size_t>(n) * 2, cudaMemcpyHostToDevice);
  } else {
    std::vector<uint16_t> tmp(static_cast<size_t>(n));
    if (t.dtype == "F32") {
      const float* p = reinterpret_cast<const float*>(src);
      for (int64_t i = 0; i < n; ++i) tmp[i] = f32_to_bf16(p[i]);
    } else {
      const uint16_t* p = reinterpret_cast<const uint16_t*>(src);
      for (int64_t i = 0; i < n; ++i) tmp[i] = f32_to_bf16(f16_to_f32(p[i]));
    }
    ce = cudaMemcpy(dst, tmp.data(), static_cast<size_t>(n) * 2, cudaMemcpyHostToDevice);
  }
  if (ce != cudaSuccess) { *err = std::string("cudaMemcpy: ") + cudaGetErrorString(ce); return B200_ERR_CUDA; }
  return 0;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

// JSON listing {"name": {"dtype": "...", "shape": [...], "bytes": n}, ...} of a checkpoint (dir, index or single file).
int64_t b200_safetensors_list(const char* path, char* buf, size_t cap) {
  if (!path) { set_error("null path"); return B200_ERR_INVALID; }
  Checkpoint ck;
  std::string err;
  if (!ck.open_path(path, &err)) { set_error("%s", err.c_str()); return B200_ERR_INVALID; }
  std::string o = "{";
  bool first = true;
  for (auto& kv : ck.index) {
    if (!first) o += ",";
    first = false;
    o += json_str(kv.first) + ":{\"dtype\":" + json_str(kv.second.second->dtype) + ",\"shape\":[";
    for (size_t i = 0; i < kv.second.second->shape.size(); ++i) o += (i ? "," : "") + std::to_string(kv.second.second->shape[i]);
    o += "],\"bytes\":" + std::to_string(kv.second.second->end - kv.second.second->begin) + "}";
  }
  o += "}";
  if (buf && cap > o.size()) memcpy(buf, o.c_str(), o.size() + 1);
  return static_cast<int64_t>(o.size());
}

// Fill the architecture fields of cfg from <dir>/config.json (HF LlamaConfig keys); other fields keep their values.
int b200_config_from_hf(const char* dir, b200_config* cfg) {
  if (!dir || !cfg) { set_error("null argument"); return B200_ERR_INVALID; }
  std::string txt;
  if (!read_text(std::string(dir) + "/config.json", &txt)) { set_error("cannot read %s/config.json", dir); return B200_ERR_NOT_FOUND; }
  JVal root;
  std::string jerr;
  if (!JParser(txt.data(), txt.size()).parse(&root, &jerr) || root.type != JVal::Obj) { set_error("config.json: %s", jerr.c_str()); return B200_ERR_INVALID; }
  auto num = [&](const char* k, double def) { const JVal* v = root.get(k); return v && v->type == JVal::Num ? v->num : def; };
  cfg->num_layers = static_cast<int>(num("num_hidden_layers", cfg->num_layers));
  cfg->hidden = static_cast<int>(num("hidden_size", cfg->hidden));
  cfg->q_heads = static_cast<int>(num("num_attention_heads", cfg->q_heads));
  cfg->kv_heads = static_cast<int>(num("num_key_value_heads", cfg->q_heads));
  cfg->intermediate = static_cast<int>(num("intermediate_size", cfg->intermediate));
  cfg->vocab = static_cast<int>(num("vocab_size", cfg->vocab));
  cfg->rms_eps = static_cast<float>(num("rms_norm_eps", cfg->rms_eps));
  double theta = num("rope_theta", cfg->rope_theta);
  if (const JVal* rp = root.get("rope_parameters")) if (const JVal* t = rp->get("rope_theta"); t && t->type == JVal::Num) theta = t->num;
  cfg->rope_theta = static_cast<float>(theta);
  // RoPE frequency scaling: HF "rope_scaling" (transformers < 5) or "rope_parameters" (>= 5); Llama-3.1/3.2 ship
  // rope_type "llama3" with factor 8 — loading those with an unscaled table would silently diverge from vLLM/HF
  cfg->rope_scaling_type = 0;
  const JVal* rs = root.get("rope_scaling");
  if (!rs || rs->type != JVal::Obj) rs = root.get("rope_parameters");
  if (rs && rs->type == JVal::Obj) {
    std::string ty = "default";
    if (const JVal* t = rs->get("rope_type"); t && t->type == JVal::Str) ty = t->str;
    else if (const JVal* t2 = rs->get("type"); t2 && t2->type == JVal::Str) ty = t2->str;
    auto rnum = [&](const char* k, double def) { const JVal* v = rs->get(k); return v && v->type == JVal::Num ? v->num : def; };
    if (ty == "default") {
    } else if (ty == "linear") {
      cfg->rope_scaling_type = 1;
      cfg->rope_factor = static_cast<float>(rnum("factor", 1.0));
    } else if (ty == "llama3") {
      cfg->rope_scaling_type = 2;
      cfg->rope_factor = static_cast<float>(rnum("factor", 8.0));
      cfg->rope_low_freq_factor = static_cast<float>(rnum("low_freq_factor", 1.0));
      cfg->rope_high_freq_factor = static_cast<float>(rnum("high_freq_factor", 4.0));
      cfg->rope_original_max_pos = static_cast<int>(rnum("original_max_position_embeddings", 8192));
    } else {
      set_error("rope scaling type \"%s\" is not supported (default, linear, llama3)", ty.c_str());
      return B200_ERR_INVALID;
    }
  }
  // the runner (vLLM's --runner auto): a base model (LlamaModel, MistralModel) has no lm_head and serves embeddings; a
  // *ForSequenceClassification model pools into its score head (vLLM's as_seq_cls_model).  Any other *For* head is refused
  // by name rather than served as whatever the runner defaults to.
  int runner = cfg->runner;
  int num_labels = cfg->num_labels, score_activation = cfg->score_activation, score_join_pair = cfg->score_join_pair;
  if (const JVal* ar = root.get("architectures"); ar && ar->type == JVal::Arr && !ar->arr.empty() && ar->arr[0].type == JVal::Str) {
    const std::string& a = ar->arr[0].str;
    auto ends_with = [&](const char* suf) { const size_t n = strlen(suf); return a.size() > n && a.compare(a.size() - n, n, suf) == 0; };
    num_labels = 0;
    score_activation = 0;
    score_join_pair = 0;
    if (a == "LlamaModel" || a == "MistralModel") {
      runner = B200_RUNNER_POOLING;
    } else if (ends_with("ForCausalLM")) {
      runner = B200_RUNNER_GENERATE;
    } else if (a == "LlamaForSequenceClassification" || a == "MistralForSequenceClassification") {
      runner = B200_RUNNER_POOLING;
      // HF PretrainedConfig: num_labels, else len(id2label), else 2
      num_labels = 2;
      if (const JVal* v = root.get("id2label"); v && v->type == JVal::Obj) num_labels = static_cast<int>(v->obj.size());
      if (const JVal* v = root.get("num_labels"); v && v->type == JVal::Num) num_labels = static_cast<int>(v->num);
      if (num_labels < 1 || num_labels > B200_MAX_SCORE_LABELS) {
        set_error("%s with %d labels is not supported: a score head has 1 to %d labels (one warp applies the activation, "
                  "lane l holding logit l)", a.c_str(), num_labels, B200_MAX_SCORE_LABELS);
        return B200_ERR_INVALID;
      }
      // vLLM's get_act_fn / PoolerClassify: problem_type picks the activation, its absence the default by label count
      if (const JVal* pt = root.get("problem_type"); pt && pt->type == JVal::Str) {
        if (pt->str == "regression") score_activation = 3;
        else if (pt->str == "single_label_classification") score_activation = num_labels == 1 ? 1 : 2;
        else if (pt->str == "multi_label_classification") score_activation = 1;
        else {
          set_error("problem_type \"%s\" is not supported (regression, single_label_classification, "
                    "multi_label_classification)", pt->str.c_str());
          return B200_ERR_INVALID;
        }
      }
      // vLLM's CrossEncoderIOProcessor: use_sep_token (default true) tokenizes (query, document) as a pair
      if (const JVal* v = root.get("use_sep_token"); v && v->type == JVal::Bool) score_join_pair = v->b ? 0 : 1;
    } else if (a.find("For") != std::string::npos) {
      set_error("architecture %s is not supported (*ForCausalLM, LlamaModel, MistralModel, LlamaForSequenceClassification, "
                "MistralForSequenceClassification)", a.c_str());
      return B200_ERR_INVALID;
    }
  }
  // architecture switches the kernels do not implement are refused, not ignored.  Mistral is the Llama block with an
  // optional sliding window, which b200_engine_create bounds max_model_len by.
  if (const JVal* mt = root.get("model_type"); mt && mt->type == JVal::Str && mt->str != "llama" && mt->str != "mistral") {
    set_error("model_type \"%s\" is not supported (llama, mistral)", mt->str.c_str());
    return B200_ERR_INVALID;
  }
  int sliding_window = 0;
  if (const JVal* sw = root.get("sliding_window"); sw && sw->type == JVal::Num) {
    if (!(sw->num >= 1 && sw->num <= 2147483647.0)) {
      set_error("sliding_window %g is not a positive integer", sw->num);
      return B200_ERR_INVALID;
    }
    sliding_window = static_cast<int>(sw->num);
  }
  // the pooling type a sentence-transformers checkpoint declares (modules.json, then <Pooling module>/config.json, as
  // vLLM's get_pooling_config reads them), checked when the checkpoint pools: none declared = last token, the only mode
  // the engine serves; any other mode, alone or beside last token, is refused
  if (runner == B200_RUNNER_POOLING) {
    std::string mods;
    JVal mroot;
    std::string merr;
    if (read_text(std::string(dir) + "/modules.json", &mods) && JParser(mods.data(), mods.size()).parse(&mroot, &merr) &&
        mroot.type == JVal::Arr) {
      for (auto& mod : mroot.arr) {
        const JVal* ty = mod.get("type");
        const JVal* path = mod.get("path");
        if (!ty || ty->type != JVal::Str || ty->str != "sentence_transformers.models.Pooling" || !path || path->type != JVal::Str) continue;
        std::string ptxt;
        JVal proot;
        if (!read_text(std::string(dir) + "/" + path->str + "/config.json", &ptxt) ||
            !JParser(ptxt.data(), ptxt.size()).parse(&proot, &merr) || proot.type != JVal::Obj)
          continue;
        for (auto& kv : proot.obj) {
          if (kv.first.rfind("pooling_mode_", 0) != 0 || kv.second.type != JVal::Bool || !kv.second.b) continue;
          const std::string mode = kv.first.substr(13);
          if (mode != "lasttoken") {
            set_error("pooling mode \"%s\" (%s/config.json) is not supported: the engine serves last-token pooling only",
                      mode.c_str(), path->str.c_str());
            return B200_ERR_INVALID;
          }
        }
      }
    }
  }
  if (const JVal* ha = root.get("hidden_act"); ha && ha->type == JVal::Str && ha->str != "silu") {
    set_error("hidden_act \"%s\" is not supported (silu)", ha->str.c_str());
    return B200_ERR_INVALID;
  }
  for (const char* k : {"attention_bias", "mlp_bias"})
    if (const JVal* bflag = root.get(k); bflag && bflag->type == JVal::Bool && bflag->b) {
      set_error("%s = true is not supported", k);
      return B200_ERR_INVALID;
    }
  if (cfg->hidden % 256 || cfg->hidden > 8192 || cfg->vocab % 8 || cfg->intermediate % 64) {
    set_error("shape not supported by the kernels (hidden %% 256 == 0 and <= 8192, vocab %% 8 == 0, intermediate %% 64 == 0)");
    return B200_ERR_INVALID;
  }
  // HF Llama takes an explicit head_dim (Llama-3.2-1B: 64 with hidden 2048 and 32 heads); hidden / q_heads otherwise
  const int head_dim = static_cast<int>(num("head_dim", cfg->q_heads ? cfg->hidden / cfg->q_heads : 0));
  if (head_dim != 64 && head_dim != 128) {
    set_error("head_dim %d is not supported (the kernels serve 64 and 128)", head_dim);
    return B200_ERR_INVALID;
  }
  if (cfg->kv_heads < 1 || cfg->q_heads % cfg->kv_heads || cfg->q_heads / cfg->kv_heads > 16) {
    set_error("GQA ratio %d:%d is not supported (kv_heads must divide q_heads, with 1 to 16 query heads per KV head)",
              cfg->q_heads, cfg->kv_heads);
    return B200_ERR_INVALID;
  }
  if ((cfg->q_heads * head_dim) % 128) {
    set_error("head_dim %d with %d query heads is not supported (q_heads * head_dim must be a multiple of 128: head_dim 64 "
              "needs an even q_heads)", head_dim, cfg->q_heads);
    return B200_ERR_INVALID;
  }
  // The head size is not a free parameter of the weights: the first layer's q / k projections have q_heads * head_dim and
  // kv_heads * head_dim rows.  A config.json that contradicts the checkpoint beside it (an edited head_dim, or a config
  // written for other weights) is refused here, before an engine of the wrong shape is built.  A directory without
  // safetensors (config only) is not checked.
  {
    Checkpoint ck;
    std::string err;
    if (ck.open_path(dir, &err)) {
      auto rows = [&](const char* name) -> int64_t {
        auto it = ck.index.find(name);
        return it == ck.index.end() || it->second.second->shape.size() != 2 ? -1 : it->second.second->shape[0];
      };
      // HF writes a *ForCausalLM's tensors under "model." and a base model's (LlamaModel, MistralModel) without it
      const char* pre = ck.index.count("model.layers.0.self_attn.q_proj.weight") ? "model." : "";
      const int64_t qr = rows((std::string(pre) + "layers.0.self_attn.q_proj.weight").c_str()),
                    kr = rows((std::string(pre) + "layers.0.self_attn.k_proj.weight").c_str());
      if ((qr >= 0 && qr != static_cast<int64_t>(cfg->q_heads) * head_dim) ||
          (kr >= 0 && kr != static_cast<int64_t>(cfg->kv_heads) * head_dim)) {
        set_error("head_dim %d does not match the checkpoint: layer 0 has q_proj / k_proj of %lld / %lld rows, not "
                  "q_heads * head_dim = %d / kv_heads * head_dim = %d", head_dim, static_cast<long long>(qr),
                  static_cast<long long>(kr), cfg->q_heads * head_dim, cfg->kv_heads * head_dim);
        return B200_ERR_INVALID;
      }
    }
  }
  cfg->head_dim = head_dim;
  cfg->runner = runner;
  cfg->sliding_window = sliding_window;
  cfg->num_labels = num_labels;
  cfg->score_activation = score_activation;
  cfg->score_join_pair = score_join_pair;
  if (const JVal* e = root.get("eos_token_id"); e && e->type == JVal::Num) cfg->eos_token_id = static_cast<int>(e->num);
  return 0;
}

// Replace the engine's (seeded random) weights with an HF Llama checkpoint.  The engine must be idle.
int b200_engine_load_safetensors(b200_engine* e, const char* path) {
  if (!e || !path) { set_error("null argument"); return B200_ERR_INVALID; }
  Checkpoint ck;
  std::string err;
  if (!ck.open_path(path, &err)) { set_error("%s", err.c_str()); return B200_ERR_INVALID; }
  auto dev = [&](const std::string& name, void** p, uint64_t* nb) { return b200_engine_tensor_info(e, name.c_str(), nb, p); };
  void* p = nullptr;
  uint64_t nb = 0;
  // shapes are recovered from the engine tensors themselves
  if (dev("final_norm", &p, &nb)) return B200_ERR_NOT_FOUND;
  const int64_t H = static_cast<int64_t>(nb / 2);
  if (dev("embed", &p, &nb)) return B200_ERR_NOT_FOUND;
  const int64_t V = static_cast<int64_t>(nb / 2) / H;
  int rc;
#define LD(hfname, row0, rows, cols) if ((rc = copy_rows(ck, hfname, p, nb, row0, rows, cols, &err))) { set_error("%s", err.c_str()); return rc; }
  // a *ForCausalLM checkpoint names its tensors "model.<name>", a base model (LlamaModel, MistralModel) "<name>"
  const std::string pre = ck.index.count("model.embed_tokens.weight") ? "model." : "";
  LD(pre + "embed_tokens.weight", 0, V, H);
  if (dev("final_norm", &p, &nb)) return B200_ERR_NOT_FOUND;
  LD(pre + "norm.weight", 0, 1, H);
  if (b200_engine_tensor_info(e, "score", &nb, &p) == 0) {   // a score head [num_labels, H], bf16 as loaded
    const int64_t labels = static_cast<int64_t>(nb / 2) / H;
    if (!ck.index.count("score.weight")) {
      set_error("missing tensor score.weight: the engine has a score head of [%lld, %lld] (num_labels = %lld)",
                static_cast<long long>(labels), static_cast<long long>(H), static_cast<long long>(labels));
      return B200_ERR_NOT_FOUND;
    }
    LD("score.weight", 0, labels, H);
  } else if (ck.index.count("score.weight") && !ck.index.count("lm_head.weight")) {
    set_error("the checkpoint has a score head (score.weight) and no lm_head.weight: a sequence-classification model is "
              "served by a pooling engine with num_labels > 0, not loaded as %s", b200_engine_tensor_info(e, "lm_head", &nb, &p) == 0 ? "a generator" : "an embedding model");
    return B200_ERR_INVALID;
  }
  if (b200_engine_tensor_info(e, "lm_head", &nb, &p) == 0) {   // a pooling engine has no lm_head
    // tie_word_embeddings: checkpoints without lm_head.weight reuse the embedding matrix
    const std::string head = ck.index.count("lm_head.weight") ? "lm_head.weight" : pre + "embed_tokens.weight";
    LD(head, 0, V, H);
  }
  for (int l = 0;; ++l) {
    const std::string ep = "layers." + std::to_string(l) + ".", hp = pre + "layers." + std::to_string(l) + ".";
    if (dev(ep + "wqkv", &p, &nb)) break;  // no more layers in the engine
    auto qit = ck.index.find(hp + "self_attn.q_proj.weight"), kit = ck.index.find(hp + "self_attn.k_proj.weight");
    if (qit == ck.index.end() || kit == ck.index.end() || qit->second.second->shape.size() != 2) { set_error("missing %sself_attn.{q,k}_proj.weight", hp.c_str()); return B200_ERR_NOT_FOUND; }
    const int64_t qrows = qit->second.second->shape[0], krows = kit->second.second->shape[0];
    LD(hp + "self_attn.q_proj.weight", 0, qrows, H);
    LD(hp + "self_attn.k_proj.weight", qrows, krows, H);
    LD(hp + "self_attn.v_proj.weight", qrows + krows, krows, H);
    if (dev(ep + "wo", &p, &nb)) return B200_ERR_NOT_FOUND;
    LD(hp + "self_attn.o_proj.weight", 0, H, qrows);
    if (dev(ep + "wgu", &p, &nb)) return B200_ERR_NOT_FOUND;
    const int64_t I = static_cast<int64_t>(nb / 2) / H / 2;
    LD(hp + "mlp.gate_proj.weight", 0, I, H);
    LD(hp + "mlp.up_proj.weight", I, I, H);
    if ((rc = engine_relayout_gate_up(e, (ep + "wgu").c_str()))) return rc;   // logical [gate | up] -> interleaved 64-row blocks
    if (dev(ep + "wdown", &p, &nb)) return B200_ERR_NOT_FOUND;
    LD(hp + "mlp.down_proj.weight", 0, H, I);
    if (dev(ep + "norm1", &p, &nb)) return B200_ERR_NOT_FOUND;
    LD(hp + "input_layernorm.weight", 0, 1, H);
    if (dev(ep + "norm2", &p, &nb)) return B200_ERR_NOT_FOUND;
    LD(hp + "post_attention_layernorm.weight", 0, 1, H);
  }
#undef LD
  return 0;
}

}  // extern "C"
