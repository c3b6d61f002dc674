// Serving shell: the reference's request path restated in C++ around the in-process engine.
//   internal/openaiserver/handler.go:20-49     route table under /openai (R1)
//   internal/modelproxy/handler.go:57-159      ServeHTTP / proxyHTTP: parse -> gauge -> pick -> serve, <=3 retries (R2, R5)
//   internal/modelproxy/request.go:45-63       error bodies {"error":"..."}\n, 5xx text hidden
//   internal/apiutils/request.go:64-225        ParseRequest: JSON body, model_adapter split, prefix (R3)
//   api/openai/v1/chat_completions.go:525-543  Prefix(n): first user message, first n runes (R4)
//   internal/metrics/metrics.go:16-27          kubeai_inference_requests_active gauge (R11)
// and the backend half the reference leaves to vLLM: tokenise + chat template, stream tokens as
// OpenAI SSE chunks in vLLM's framing (api/openai/v1/reference/example-requests.vllm.output:139-160;
// vllm/entrypoints/openai/chat_completion/serving.py) (K12, K13).
// The HTTP hop of proxyHTTP (handler.go:116-158) is replaced by b200_submit_n/b200_wait_any/b200_poll.
#include <arpa/inet.h>
#include <errno.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <signal.h>
#include <sys/socket.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <map>
#include <mutex>
#include <random>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "../../include/b200engine.h"
#include "errors.h"
#include "hostutil.h"
#include "tokenizer.h"

namespace b200 {

struct Server {
  std::string model;
  std::set<std::string> adapters;
  int strategy = B200_LB_LEAST_LOAD;
  int mean_load_pct = 125, replication = 256, prefix_chars = 100;
  int max_retries = 3;
  int default_max_tokens = 256;
  std::vector<b200_engine*> replicas;
  std::vector<std::string> addrs;  // "gpu:<i>"
  b200_router* router = nullptr;
  Tokenizer tok;
  int max_model_len = 2048;
  bool sampling = false;   // b200_server_config.enable_sampling: serve temperature >= 1e-5 (else greedy only)
  bool logprobs = false;   // b200_server_config.enable_logprobs: serve logprobs / top_logprobs (else a 400)
  bool edits = false;      // b200_server_config.enable_logits_processors: serve penalties, min_p, min_tokens, logit_bias
  bool prompt_lp = false;  // b200_server_config.enable_prompt_logprobs: serve prompt_logprobs and completions echo
  int max_n = 0;           // b200_server_config.max_n: >= 2 serves n up to it (else n > 1 is a 400)
  bool pooling = false;    // the replicas run the pooling runner: /v1/embeddings is served, the generation routes are not
  int hidden = 0;          // embedding size (pooling)
  // the replicas' score head (b200_config.num_labels > 0): /v1/rerank is served, /v1/embeddings and generation are not;
  // join_pair: b200_config.score_join_pair (pairs tokenized as query + document through the single template)
  int num_labels = 0;
  bool join_pair = false;
  // optional real tokenizer (b200_server_set_tokenizer): a checkpoint's tokenizer.json instead of the synthetic byte/word ids
  const b200_tokenizer* real_tok = nullptr;

  std::mutex mmu;
  std::map<std::string, int64_t> active;  // kubeai_inference_requests_active{request_model=...}
  std::atomic<int64_t> requests_total{0}, retries_total{0}, errors_total{0};
  std::vector<std::unique_ptr<std::atomic<int>>> faults;  // fault injection: fail the next N submits on replica i

  // HTTP listener
  int listen_fd = -1;
  std::thread acceptor;
  std::atomic<bool> stopping{false};
  std::atomic<int> live_conns{0};
  std::mutex conn_mu;
  std::set<int> conn_fds;          // open client sockets: shut down by the destructor so no thread outlives the Server
  static constexpr int kMaxConns = 4096;
  static constexpr int kIdleTimeoutS = 60;  // keep-alive read timeout (SO_RCVTIMEO)

  // replicas whose engine reported a fatal error are taken out of the endpoint set, as reconcileEndpoints drops
  // endpoints that vanished (internal/loadbalancer/group.go:119-131)
  std::mutex dead_mu;
  std::vector<char> dead;
  std::string adapters_csv;
  void drop_replica(int i);

  ~Server() {
    stopping = true;
    if (listen_fd >= 0) {
      shutdown(listen_fd, SHUT_RDWR);
      close(listen_fd);
    }
    if (acceptor.joinable()) acceptor.join();
    {
      // wake every connection thread blocked in recv()/send(); each closes its own fd and leaves
      std::lock_guard<std::mutex> lk(conn_mu);
      for (int fd : conn_fds) shutdown(fd, SHUT_RDWR);
    }
    while (live_conns.load() > 0) usleep(1000);
    if (router) b200_router_destroy(router);
  }
};

void Server::drop_replica(int i) {
  std::lock_guard<std::mutex> lk(dead_mu);
  if (i < 0 || i >= static_cast<int>(dead.size()) || dead[i]) return;
  dead[i] = 1;
  std::vector<std::string> names;
  std::vector<const char*> np, ap, dp;
  for (size_t k = 0; k < replicas.size(); ++k) {
    if (dead[k]) continue;
    names.push_back("gpu-" + std::to_string(k));
  }
  size_t j = 0;
  for (size_t k = 0; k < replicas.size(); ++k) {
    if (dead[k]) continue;
    np.push_back(names[j++].c_str());
    ap.push_back(addrs[k].c_str());
    dp.push_back(adapters_csv.c_str());
  }
  b200_router_set_endpoints(router, np.data(), ap.data(), dp.data(), static_cast<int32_t>(np.size()));
}

namespace {

std::string hex_id(int n) {
  static thread_local std::mt19937_64 rng{std::random_device{}()};
  static const char* h = "0123456789abcdef";
  std::string s;
  for (int i = 0; i < n; ++i) s += h[rng() & 15];
  return s;
}

struct Writer {
  const b200_response_writer* w;
  bool begun = false;
  bool gone = false;
  void begin(int status, const char* ctype) {
    if (begun) return;
    begun = true;
    if (w->begin && w->begin(w->ud, status, ctype)) gone = true;
  }
  void write(const std::string& s) {
    if (gone || !w->write) return;
    if (w->write(w->ud, s.data(), s.size())) gone = true;
  }
};

// modelproxy/request.go:45-63 sendErrorResponse
int send_error(Writer& w, int status, const std::string& msg) {
  static const std::map<int, const char*> text = {{500, "Internal Server Error"}, {502, "Bad Gateway"},
                                                  {503, "Service Unavailable"}, {504, "Gateway Timeout"}};
  std::string m = msg;
  if (status >= 500) {
    auto it = text.find(status);
    m = it == text.end() ? "Internal Server Error" : it->second;
  }
  w.begin(status, "application/json");
  w.write("{\"error\":" + json_str(m) + "}\n");
  return status;
}

struct ParsedRequest {
  bool chat = true;
  bool embed = false;   // /v1/embeddings (the reference's EmbeddingRequest: no Prefix)
  bool rerank = false;  // /v1/rerank on a score-head server (the reference's RerankRequest: no Prefix)
  std::string requested_model, model, adapter, prefix;
  std::vector<std::pair<std::string, std::string>> messages;
  std::vector<int32_t> prompt_ids;  // completions with token-id prompt
  std::string prompt_text;
  bool prompt_is_ids = false;
  int max_tokens = -1;
  bool stream = false, include_usage = false, ignore_eos = false;
  double temperature = 0.0;   // absent = greedy
  double top_p = 1.0;
  int top_k = 0;
  bool has_seed = false;
  int64_t seed = 0;
  int logprobs = -1;   // -1: none; else the number of most likely tokens per position (chat top_logprobs, completions logprobs)
  // read only when the server serves them: prompt_logprobs (-1: absent) and completions echo
  int prompt_logprobs = -1;
  bool echo = false;
  int n = 1;   // choices (parallel sampling), read only when the server serves n
  std::vector<int32_t> stop_ids;
  // logits edits (b200_sampling): read only when the server serves them
  double presence = 0.0, frequency = 0.0, repetition = 1.0, min_p = 0.0;
  int min_tokens = 0;
  std::vector<int32_t> bias_ids;
  std::vector<float> bias_values;
};

std::string content_text(const JVal& c) {
  if (c.type == JVal::Str) return c.str;
  std::string s;
  if (c.type == JVal::Arr)
    for (auto& part : c.arr) {
      const JVal* t = part.get("text");
      if (t && t->type == JVal::Str) s += t->str;
    }
  return s;  // content:null -> "" (the reference nil-derefs here, chat_completions.go:532; not copied)
}

// apiutils.ParseRequest for the JSON branch.  Returns 0 or an HTTP status with *err set.
int parse_request(Server& sv, const std::string& path, const std::string& ctype, const char* body, size_t len,
                  ParsedRequest* pr, std::string* err) {
  std::string media = ctype.substr(0, ctype.find(';'));
  while (!media.empty() && media.back() == ' ') media.pop_back();
  for (auto& ch : media) ch = static_cast<char>(tolower(ch));
  if (media == "multipart/form-data") {
    *err = "bad request: reading multipart form data: not supported by this engine (speech routes are out of scope)";
    return 400;
  }
  if (path == "/v1/chat/completions") pr->chat = true;
  else if (path == "/v1/completions") pr->chat = false;
  else if (path == "/v1/embeddings") pr->embed = true;
  else if (path == "/v1/rerank" && sv.num_labels > 0) pr->rerank = true;
  else {
    *err = "bad request: reading model from body: unknown path: \"" + path + "\"";
    return 400;
  }
  JVal root;
  std::string jerr;
  if (!JParser(body, len).parse(&root, &jerr) || root.type != JVal::Obj) {
    *err = "bad request: reading model from body: decoding: " + (jerr.empty() ? std::string("expected JSON object") : jerr);
    return 400;
  }
  if (pr->rerank) {
    // RerankRequest's typed fields, as Go decodes them (api/openai/v1/rerank.go): query a string, documents a list of
    // strings, top_n an integer; null leaves a field at its zero value
    auto type_name = [](const JVal& v) {
      switch (v.type) {
        case JVal::Bool: return "boolean";
        case JVal::Num: return "number";
        case JVal::Str: return "string";
        case JVal::Arr: return "array";
        case JVal::Obj: return "object";
        default: return "null";
      }
    };
    auto decoding = [&](const JVal& v, const char* go_type, const std::string& where) {
      *err = std::string("bad request: reading model from body: decoding: json: cannot unmarshal JSON ") + type_name(v) +
             " into Go " + go_type + " within \"" + where + "\"";
      return 400;
    };
    if (const JVal* q = root.get("query"); q && q->type != JVal::Null && q->type != JVal::Str) return decoding(*q, "string", "/query");
    if (const JVal* d = root.get("documents"); d && d->type != JVal::Null) {
      if (d->type != JVal::Arr) return decoding(*d, "[]string", "/documents");
      for (size_t i = 0; i < d->arr.size(); ++i)
        if (d->arr[i].type != JVal::Str && d->arr[i].type != JVal::Null) return decoding(d->arr[i], "string", "/documents/" + std::to_string(i));
    }
    if (const JVal* t = root.get("top_n"); t && t->type != JVal::Null &&
        (t->type != JVal::Num || t->num != std::floor(t->num) || std::fabs(t->num) > 9.2e18))
      return decoding(*t, "int", "/top_n");
  }
  const JVal* m = root.get("model");
  if (!m || m->type != JVal::Str || m->str.empty()) {
    *err = "bad request: reading model from body: missing 'model' field";
    return 400;
  }
  pr->requested_model = m->str;
  // apiutils/model.go:23-29 SplitModelAdapter: first "_"
  size_t us = m->str.find('_');
  pr->model = m->str.substr(0, us);
  pr->adapter = us == std::string::npos ? "" : m->str.substr(us + 1);
  // LookupModel (modelclient/client.go:27-64): nil -> ErrModelNotFound
  if (pr->model != sv.model || (!pr->adapter.empty() && !sv.adapters.count(pr->adapter))) {
    *err = "model not found: \"" + pr->requested_model + "\"";
    return 404;
  }
  if (pr->embed || pr->rerank) return 0;   // their fields are read by serve_embeddings / serve_rerank
  if (pr->chat) {
    const JVal* msgs = root.get("messages");
    if (msgs && msgs->type == JVal::Arr) {
      for (auto& mm : msgs->arr) {
        const JVal* role = mm.get("role");
        const JVal* content = mm.get("content");
        pr->messages.emplace_back(role && role->type == JVal::Str ? role->str : "", content ? content_text(*content) : "");
      }
    }
    for (auto& mm : pr->messages)
      if (mm.first == "user") {
        pr->prefix = mm.second;
        break;
      }
  } else {
    const JVal* p = root.get("prompt");
    if (p && p->type == JVal::Str) {
      pr->prompt_text = p->str;
      pr->prefix = p->str;
    } else if (p && p->type == JVal::Arr && !p->arr.empty()) {
      const JVal& first = p->arr[0];
      if (first.type == JVal::Str) {
        pr->prompt_text = first.str;
        pr->prefix = first.str;
      } else if (first.type == JVal::Num) {
        pr->prompt_is_ids = true;
        for (auto& e : p->arr) pr->prompt_ids.push_back(static_cast<int32_t>(e.num));
      } else if (first.type == JVal::Arr) {
        pr->prompt_is_ids = true;
        for (auto& e : first.arr) pr->prompt_ids.push_back(static_cast<int32_t>(e.num));
      }
    }
  }
  // r.Prefix only under PrefixHash (apiutils/request.go:219-223)
  pr->prefix = sv.strategy == B200_LB_PREFIX_HASH ? first_n_runes(pr->prefix, sv.prefix_chars) : "";  // firstNChars (utils.go:5-8)
  if (const JVal* v = root.get("max_completion_tokens"); v && v->type == JVal::Num) pr->max_tokens = static_cast<int>(v->num);
  if (const JVal* v = root.get("max_tokens"); v && v->type == JVal::Num) pr->max_tokens = static_cast<int>(v->num);
  if (const JVal* v = root.get("stream"); v && v->type == JVal::Bool) pr->stream = v->b;
  if (const JVal* so = root.get("stream_options"))
    if (const JVal* iu = so->get("include_usage"); iu && iu->type == JVal::Bool) pr->include_usage = iu->b;
  if (const JVal* v = root.get("ignore_eos"); v && v->type == JVal::Bool) pr->ignore_eos = v->b;
  // sampling (vLLM's request fields; top_k is its extension).  The JSON numbers are doubles: an integer field that is not
  // an exact integer, or a seed beyond 2^53, is refused rather than rounded.
  const char* bad_sampling = nullptr;
  if (const JVal* v = root.get("temperature"); v && v->type == JVal::Num) {
    pr->temperature = v->num;
    if (!(v->num >= 0 && v->num <= 3.0e38)) bad_sampling = "temperature must be a finite number >= 0";   // finite as a float too
  }
  if (const JVal* v = root.get("top_p"); v && v->type == JVal::Num) {
    pr->top_p = v->num;
    if (!(v->num > 0 && v->num <= 1)) bad_sampling = "top_p must be in (0, 1]";
  }
  if (const JVal* v = root.get("top_k"); v && v->type == JVal::Num) {
    if (!(v->num >= -1 && v->num == std::floor(v->num) && v->num <= 2147483647.0)) bad_sampling = "top_k must be an integer >= -1";
    else pr->top_k = static_cast<int>(v->num);
  }
  if (const JVal* v = root.get("seed"); v && v->type == JVal::Num) {
    if (!(v->num == std::floor(v->num) && std::fabs(v->num) <= 9007199254740992.0)) bad_sampling = "seed must be an integer of magnitude <= 2^53";
    else {
      pr->seed = static_cast<int64_t>(v->num);
      pr->has_seed = true;
    }
  }
  if (bad_sampling) {
    *err = std::string("bad request: ") + bad_sampling;
    return 400;
  }
  if (sv.logprobs) {
    // chat: "logprobs": bool, "top_logprobs": 0..20 (> 0 needs logprobs, vLLM chat_completion/protocol.py); completions:
    // "logprobs": 0..20.  null is absent; anything else that is not an integer in range is refused.
    const char* bad_lp = nullptr;
    auto count = [&](const JVal* v, const char* msg) {
      if (!v || v->type == JVal::Null) return -1;
      if (v->type != JVal::Num || !(v->num >= 0 && v->num <= B200_MAX_LOGPROBS && v->num == std::floor(v->num))) {
        bad_lp = msg;
        return -1;
      }
      return static_cast<int>(v->num);
    };
    const JVal* lp = root.get("logprobs");
    if (pr->chat) {
      bool on = false;
      if (lp && lp->type == JVal::Bool) on = lp->b;
      else if (lp && lp->type != JVal::Null) bad_lp = "logprobs must be a boolean";
      const int n = count(root.get("top_logprobs"), "top_logprobs must be an integer in 0..20");
      if (!bad_lp && n > 0 && !on) bad_lp = "top_logprobs needs \"logprobs\": true";
      if (on) pr->logprobs = n > 0 ? n : 0;
    } else {
      pr->logprobs = count(lp, "logprobs must be an integer in 0..20");
    }
    if (bad_lp) {
      *err = std::string("bad request: ") + bad_lp;
      return 400;
    }
  }
  if (sv.prompt_lp) {
    // vLLM's checks, in its order (CompletionRequest / ChatCompletionRequest check_logprobs, then SamplingParams
    // _validate_logprobs at max_logprobs 20); null is absent.  Chat echo keeps its 400 below: it means something else there.
    std::string bad_plp;
    if (const JVal* v = root.get("prompt_logprobs"); v && v->type != JVal::Null) {
      if (v->type != JVal::Num || v->num != std::floor(v->num) || std::fabs(v->num) > 2147483647.0) {
        bad_plp = "prompt_logprobs must be an integer";
      } else {
        const int n = static_cast<int>(v->num);
        if (pr->stream && (n > 0 || n == -1)) bad_plp = "`prompt_logprobs` are not available when `stream=True`.";
        else if (n < 0 && n != -1) bad_plp = "`prompt_logprobs` must be a positive value or -1.";
        else if (n == -1 || n > B200_MAX_LOGPROBS)
          bad_plp = "Requested prompt logprobs of " + std::to_string(n == -1 ? sv.tok.vocab : n) + ", which is greater than max allowed: " +
                    std::to_string(B200_MAX_LOGPROBS);
        else pr->prompt_logprobs = n;
      }
    }
    if (const JVal* v = root.get("echo"); !pr->chat && v && v->type == JVal::Bool) pr->echo = v->b;
    if (!bad_plp.empty()) {
      *err = "bad request: " + bad_plp;
      return 400;
    }
  }
  if (sv.edits) {
    // vLLM's SamplingParams ranges (sampling_params.py _verify_args, _validate_logit_bias); null is absent
    std::string bad_ed;
    auto number = [&](const char* k, double* dst, double lo, double hi, bool lo_open) {
      const JVal* v = root.get(k);
      if (!v || v->type == JVal::Null || !bad_ed.empty()) return;
      if (v->type != JVal::Num) { bad_ed = std::string(k) + " must be a number"; return; }
      char b[160];
      if (!((lo_open ? v->num > lo : v->num >= lo) && v->num <= hi)) {
        if (hi > 1e30) snprintf(b, sizeof(b), "%s must be greater than zero, got %g.", k, v->num);
        else snprintf(b, sizeof(b), "%s must be in [%g, %g], got %g.", k, lo, hi, v->num);
        bad_ed = b;
        return;
      }
      *dst = v->num;
    };
    number("presence_penalty", &pr->presence, -2.0, 2.0, false);
    number("frequency_penalty", &pr->frequency, -2.0, 2.0, false);
    number("repetition_penalty", &pr->repetition, 0.0, 3.0e38, true);
    number("min_p", &pr->min_p, 0.0, 1.0, false);
    if (const JVal* v = root.get("min_tokens"); bad_ed.empty() && v && v->type != JVal::Null) {
      if (v->type != JVal::Num || !(v->num >= 0 && v->num == std::floor(v->num) && v->num <= 2147483647.0))
        bad_ed = "min_tokens must be an integer >= 0";
      else pr->min_tokens = static_cast<int>(v->num);
    }
    if (const JVal* v = root.get("logit_bias"); bad_ed.empty() && v && v->type != JVal::Null) {
      if (v->type != JVal::Obj) bad_ed = "logit_bias must be an object of token ids to numbers";
      else if (v->obj.size() > B200_MAX_LOGIT_BIAS) bad_ed = "logit_bias takes at most " + std::to_string(B200_MAX_LOGIT_BIAS) + " entries";
      std::string oov;
      for (auto& kv : v->obj) {
        if (!bad_ed.empty()) break;
        const std::string& key = kv.first;
        size_t i = (!key.empty() && (key[0] == '-' || key[0] == '+')) ? 1 : 0;
        bool digits = i < key.size() && key.size() - i <= 9;
        for (size_t j = i; j < key.size() && digits; ++j) digits = key[j] >= '0' && key[j] <= '9';
        if (!digits) { bad_ed = "logit_bias keys must be integer token ids, got \"" + key + "\""; break; }
        if (kv.second.type != JVal::Num) { bad_ed = "logit_bias values must be numbers"; break; }
        const long id = strtol(key.c_str(), nullptr, 10);
        if (id < 0 || id >= sv.tok.vocab) { oov += (oov.empty() ? "" : ", ") + std::to_string(id); continue; }
        pr->bias_ids.push_back(static_cast<int32_t>(id));
        pr->bias_values.push_back(static_cast<float>(std::min(100.0, std::max(-100.0, kv.second.num))));   // OpenAI's clamp
      }
      if (bad_ed.empty() && !oov.empty())
        bad_ed = "token_id(s) [" + oov + "] in logit_bias contain out-of-vocab token ids. Vocabulary size: " + std::to_string(sv.tok.vocab);
    }
    if (!bad_ed.empty()) {
      *err = "bad request: " + bad_ed;
      return 400;
    }
  }
  if (sv.max_n >= 2) {
    // vLLM's SamplingParams checks of n (_verify_args, then _verify_greedy_sampling); every choice runs at once, so the
    // server's max_n bounds it.  null is absent.
    std::string bad_n;
    if (const JVal* v = root.get("n"); v && v->type != JVal::Null) {
      if (v->type != JVal::Num || v->num != std::floor(v->num) || std::fabs(v->num) > 2147483647.0) {
        bad_n = "n must be an integer";
      } else {
        const int k = static_cast<int>(v->num);
        if (k < 1) bad_n = "n must be at least 1, got " + std::to_string(k) + ".";
        else if (k > sv.max_n) bad_n = "n must be at most " + std::to_string(sv.max_n) + ", got " + std::to_string(k) + ".";
        else if (k > 1 && pr->temperature < 1e-5) bad_n = "n must be 1 when using greedy sampling, got " + std::to_string(k) + ".";
        else pr->n = k;
      }
    }
    if (!bad_n.empty()) {
      *err = "bad request: " + bad_n;
      return 400;
    }
  }
  if (const JVal* v = root.get("stop_token_ids"); v && v->type == JVal::Arr)
    for (auto& e : v->arr)
      if (e.type == JVal::Num) pr->stop_ids.push_back(static_cast<int32_t>(e.num));
  // Fields of the reference's request schema (api/openai/v1/chat_completions.go:361-470, completions.go:19-130) whose
  // semantics this engine does not implement are refused, never silently dropped.
  auto num_of = [&](const char* k, double def) { const JVal* v = root.get(k); return v && v->type == JVal::Num ? v->num : def; };
  auto truthy = [&](const char* k) {
    const JVal* v = root.get(k);
    return v && ((v->type == JVal::Bool && v->b) || (v->type == JVal::Num && v->num > 0));
  };
  auto nonempty = [&](const char* k) {
    const JVal* v = root.get(k);
    return v && ((v->type == JVal::Str && !v->str.empty()) || (v->type == JVal::Arr && !v->arr.empty()) ||
                 (v->type == JVal::Obj && !v->obj.empty()));
  };
  const char* bad = nullptr;
  if (sv.max_n < 2 && num_of("n", 1) > 1) bad = "n > 1";
  else if (num_of("best_of", 1) > 1) bad = "best_of > 1";
  else if (!sv.logprobs && (truthy("logprobs") || truthy("top_logprobs") || (!sv.prompt_lp && truthy("prompt_logprobs")))) bad = "logprobs";
  else if (!sv.prompt_lp && truthy("prompt_logprobs")) bad = "prompt_logprobs";
  else if (!pr->chat && truthy("top_logprobs")) bad = "top_logprobs on completions (use logprobs)";
  else if (nonempty("stop")) bad = "stop strings (use stop_token_ids)";
  else if ((pr->chat || !sv.prompt_lp) && truthy("echo")) bad = "echo";
  else if (nonempty("suffix")) bad = "suffix";
  else if (!sv.edits && (num_of("presence_penalty", 0) != 0 || num_of("frequency_penalty", 0) != 0 || num_of("repetition_penalty", 1) != 1)) bad = "sampling penalties";
  else if (!sv.edits && nonempty("logit_bias")) bad = "logit_bias";
  else if (nonempty("tools") || nonempty("functions")) bad = "tool calling";
  else if (!sv.edits && truthy("min_tokens")) bad = "min_tokens";
  else if (!sv.edits && num_of("min_p", 0) > 0 && pr->temperature >= 1e-5) bad = "min_p";   // harmless under greedy decoding only
  else if (const JVal* rf = root.get("response_format"); rf && rf->type == JVal::Obj) {
    const JVal* ty = rf->get("type");
    if (ty && ty->type == JVal::Str && ty->str != "text") bad = "response_format other than text";
  }
  if (bad) {
    *err = std::string("bad request: ") + bad + " is not supported by this engine";
    return 400;
  }
  return 0;
}

std::string usage_json(const b200_usage& u) {
  char b[256];
  snprintf(b, sizeof(b),
           "{\"prompt_tokens\":%d,\"total_tokens\":%d,\"completion_tokens\":%d,\"prompt_tokens_details\":{\"cached_tokens\":%d}}",
           u.prompt_tokens, u.prompt_tokens + u.completion_tokens, u.completion_tokens, u.cached_tokens);
  return b;
}

const char* finish_str(int code) { return code == B200_FINISH_STOP ? "stop" : code == B200_FINISH_LENGTH ? "length" : "abort"; }

// ---- logprobs in vLLM 0.22's OpenAI format (vllm/v1/engine/logprobs.py, chat_completion/serving.py _create_chat_logprobs,
// completion/serving.py _create_completion_logprobs)
struct LpRecord {
  int32_t id;
  float lp;
  std::vector<std::pair<int32_t, float>> top;   // the request's N most likely tokens
  bool none = false;   // the first prompt position of an echo: no record (null entries)
  int32_t rank = 0;    // prompt records: the token's rank
};

// the shortest decimal that reads back as the same fp32, after vLLM's clamp at -9999.0
std::string lp_num(float v) {
  v = std::max(v, -9999.0f);
  char b[32];
  for (int p = 6; p <= 9; ++p) {
    snprintf(b, sizeof(b), "%.*g", p, static_cast<double>(v));
    if (strtof(b, nullptr) == v) break;
  }
  return b;
}

// code points in valid UTF-8 (Python's len of the str)
size_t utf8_len(const std::string& s) {
  size_t n = 0;
  for (unsigned char c : s) n += (c & 0xC0) != 0x80;
  return n;
}

// vLLM's entries of one position: the sampled token first, then the top N without it
std::vector<std::pair<int32_t, float>> lp_entries(const LpRecord& r) {
  std::vector<std::pair<int32_t, float>> e{{r.id, r.lp}};
  for (auto& t : r.top)
    if (t.first != r.id) e.push_back(t);
  return e;
}

std::string chat_lp_item(const std::string& tok, float lp, bool with_top) {
  std::string o = "{\"token\":" + json_str(tok) + ",\"logprob\":" + lp_num(lp) + ",\"bytes\":[";
  for (size_t i = 0; i < tok.size(); ++i) o += (i ? "," : "") + std::to_string(static_cast<unsigned char>(tok[i]));
  o += "]";
  if (!with_top) o += "}";
  return o;
}

// one element of chat "logprobs.content": the token, then the first N entries
template <class Str>
std::string chat_lp_content(const LpRecord& r, const Str& token_str) {
  const auto e = lp_entries(r);
  std::string o = chat_lp_item(token_str(r.id), r.lp, true) + ",\"top_logprobs\":[";
  for (size_t j = 0; j < r.top.size() && j < e.size(); ++j) o += (j ? "," : "") + chat_lp_item(token_str(e[j].first), e[j].second, false);
  return o + "]}";
}

// completions "logprobs" of consecutive tokens, text_offset counted from `offset`: the first N + 1 entries of each position
// as a {token string: logprob} object (a string that repeats keeps its first place and takes the later value, as a dict).
// An echoed prompt's first position has null entries.
template <class Str>
std::string completion_lp(const std::vector<LpRecord>& rs, size_t offset, const Str& token_str, int n) {
  std::string off = "[", lps = "[", toks = "[", tops = "[";
  for (size_t k = 0; k < rs.size(); ++k) {
    const std::string s = token_str(rs[k].id);
    const char* sep = k ? "," : "";
    off += sep + std::to_string(offset);
    offset += utf8_len(s);
    toks += sep + json_str(s);
    if (rs[k].none) {
      lps += sep + std::string("null");
      tops += sep + std::string("null");
      continue;
    }
    lps += sep + lp_num(rs[k].lp);
    const auto e = lp_entries(rs[k]);
    std::vector<std::pair<std::string, float>> d;
    for (size_t j = 0; j <= static_cast<size_t>(n) && j < e.size(); ++j) {
      std::string key = token_str(e[j].first);
      auto it = std::find_if(d.begin(), d.end(), [&](const std::pair<std::string, float>& x) { return x.first == key; });
      if (it != d.end()) it->second = e[j].second;
      else d.emplace_back(std::move(key), e[j].second);
    }
    tops += sep + std::string("{");
    for (size_t j = 0; j < d.size(); ++j) tops += (j ? "," : "") + json_str(d[j].first) + ":" + lp_num(d[j].second);
    tops += "}";
  }
  return "{\"text_offset\":" + off + "],\"token_logprobs\":" + lps + "],\"tokens\":" + toks + "],\"top_logprobs\":" + tops + "]}";
}

// vLLM's "prompt_logprobs" list: null for the first prompt position, then per position a {"<id>": {logprob, rank,
// decoded_token}} object built as vllm/logprobs.py append_logprobs_for_next_position does (the prompt token with its rank
// first, then the top N with ranks 1..N, a repeated id keeping its first place and taking the later entry); -inf is -9999
// (clamp_prompt_logprobs)
template <class Str>
std::string prompt_lp_json(const std::vector<LpRecord>& rs, const Str& token_str) {
  auto num = [](float v) { return std::isinf(v) && v < 0 ? std::string("-9999.0") : lp_num(v); };
  std::string o = "[null";
  for (const LpRecord& r : rs) {
    struct E { int32_t id; float lp; int32_t rank; };
    std::vector<E> d{{r.id, r.lp, r.rank}};
    for (size_t j = 0; j < r.top.size(); ++j) {
      const E e{r.top[j].first, r.top[j].second, static_cast<int32_t>(j + 1)};
      auto it = std::find_if(d.begin(), d.end(), [&](const E& x) { return x.id == e.id; });
      if (it != d.end()) *it = e;
      else d.push_back(e);
    }
    o += ",{";
    for (size_t j = 0; j < d.size(); ++j)
      o += (j ? ",\"" : "\"") + std::to_string(d[j].id) + "\":{\"logprob\":" + num(d[j].lp) + ",\"rank\":" + std::to_string(d[j].rank) +
           ",\"decoded_token\":" + json_str(token_str(d[j].id)) + "}";
    o += "}";
  }
  return o + "]";
}

}  // namespace

// modelproxy.Handler.ServeHTTP + proxyHTTP with the engine in place of the reverse proxy.
// K13: the ids the backend would see for this request.  With a real tokenizer attached: the Llama-3 chat framing for chat
// requests, <|begin_of_text|> + the encoded text for completions (what the reference's vLLM pod does with the checkpoint's
// tokenizer.json and chat_template); otherwise the synthetic tokenizer and ChatML of hostutil.h.
static void render_prompt(const Server& sv, const ParsedRequest& pr, std::vector<int32_t>* ids) {
  if (pr.prompt_is_ids && !pr.chat) {
    *ids = pr.prompt_ids;
  } else if (sv.real_tok) {
    std::vector<int32_t> buf(1024);
    int64_t n = 0;
    if (pr.chat) {
      std::vector<const char*> roles, contents;
      for (auto& m : pr.messages) { roles.push_back(m.first.c_str()); contents.push_back(m.second.c_str()); }
      const bool gen = pr.messages.empty() || pr.messages.back().first != "assistant";
      n = b200_tokenizer_chat_llama3(sv.real_tok, roles.data(), contents.data(), static_cast<int>(roles.size()), gen ? 1 : 0, buf.data(), buf.size());
      if (n > static_cast<int64_t>(buf.size())) {
        buf.resize(static_cast<size_t>(n));
        n = b200_tokenizer_chat_llama3(sv.real_tok, roles.data(), contents.data(), static_cast<int>(roles.size()), gen ? 1 : 0, buf.data(), buf.size());
      }
      if (n > 0) ids->assign(buf.begin(), buf.begin() + n);
    } else {
      if (tokenizer_bos(sv.real_tok) >= 0) ids->push_back(tokenizer_bos(sv.real_tok));
      n = b200_tokenizer_encode(sv.real_tok, pr.prompt_text.data(), pr.prompt_text.size(), 1, buf.data(), buf.size());
      if (n > static_cast<int64_t>(buf.size())) {
        buf.resize(static_cast<size_t>(n));
        n = b200_tokenizer_encode(sv.real_tok, pr.prompt_text.data(), pr.prompt_text.size(), 1, buf.data(), buf.size());
      }
      if (n > 0) ids->insert(ids->end(), buf.begin(), buf.begin() + n);
    }
  } else if (pr.chat) {
    sv.tok.chat_prompt(pr.messages, ids);
  } else {
    sv.tok.encode(pr.prompt_text, ids);
  }
  if (ids->empty()) ids->push_back(sv.real_tok && tokenizer_bos(sv.real_tok) >= 0 ? tokenizer_bos(sv.real_tok) : sv.tok.im_start());
}

static int serve_inference(Server& sv, const std::string& path, const std::string& ctype, const char* body,
                           size_t len, Writer& w) {
  ParsedRequest pr;
  std::string err;
  if (int st = parse_request(sv, path, ctype, body, len, &pr, &err)) return send_error(w, st, err);
  if (!sv.sampling && pr.temperature >= 1e-5) {
    // a greedy-only server (enable_sampling 0) refuses rather than silently decoding greedily
    return send_error(w, 400, "bad request: only greedy sampling is enabled on this server: set \"temperature\": 0");
  }
  // tokenise (K13)
  std::vector<int32_t> ids;
  render_prompt(sv, pr, &ids);
  for (auto t : ids)
    if (t < 0 || t >= sv.tok.vocab) return send_error(w, 400, "bad request: prompt token id out of range");
  int max_tokens = pr.max_tokens > 0 ? pr.max_tokens : sv.default_max_tokens;
  // echo with max_tokens 0 returns the prompt only; vLLM generates one token for it and drops it (completion/protocol.py
  // to_sampling_params), and counts that token in the usage
  const bool echo_only = pr.echo && pr.max_tokens == 0;
  if (echo_only) max_tokens = 1;
  if (static_cast<int>(ids.size()) + 1 > sv.max_model_len)
    return send_error(w, 400, "bad request: prompt is longer than the model's context length");
  max_tokens = std::min(max_tokens, sv.max_model_len - static_cast<int>(ids.size()));
  if (pr.min_tokens > max_tokens)
    return send_error(w, 400, "bad request: min_tokens must be less than or equal to max_tokens=" + std::to_string(max_tokens) +
                                  ", got " + std::to_string(pr.min_tokens) + ".");

  // metrics.InferenceRequestsActive +1 / defer -1 (handler.go:76-81)
  {
    std::lock_guard<std::mutex> lk(sv.mmu);
    ++sv.active[pr.requested_model];
  }
  sv.requests_total.fetch_add(1);
  struct Dec {
    Server& s;
    std::string m;
    ~Dec() {
      std::lock_guard<std::mutex> lk(s.mmu);
      --s.active[m];
    }
  } dec{sv, pr.requested_model};

  // prompt logprobs: asked for, or echo with logprobs (which then covers the prompt with the same N)
  const int plp_n = pr.prompt_logprobs >= 0 ? pr.prompt_logprobs : (pr.echo && pr.logprobs >= 0 ? pr.logprobs : -1);
  // the echoed prompt text: the request's own text, or the decoded ids of a token-id prompt
  std::string echo_text;
  if (pr.echo && !pr.prompt_is_ids) {
    echo_text = pr.prompt_text;
  } else if (pr.echo && sv.real_tok) {
    DetokStream d;
    d.tok = sv.real_tok;
    for (auto t : ids) echo_text += d.push(t);
    echo_text += d.flush();
  } else if (pr.echo) {
    for (auto t : ids) echo_text += sv.tok.piece(t);
  }

  const std::string id = (pr.chat ? "chatcmpl-" : "cmpl-") + hex_id(32);
  const long created = static_cast<long>(time(nullptr));
  const std::string head = "{\"id\":\"" + id + "\",\"object\":\"" + (pr.chat ? "chat.completion.chunk" : "text_completion") +
                           "\",\"created\":" + std::to_string(created) + ",\"model\":" + json_str(pr.requested_model);

  // proxyHTTP (handler.go:96-159): pick an endpoint, serve, retry with a fresh pick on failure;
  // the in-flight count of every attempt is released when the request ends.
  std::vector<uint64_t> tokens_held;
  auto release_all = [&] {
    for (auto t : tokens_held) b200_router_done(sv.router, t);
    tokens_held.clear();
  };
  for (int attempt = 0;; ++attempt) {
    char addr[64];
    uint64_t ep_token = 0;
    int rc = b200_router_pick(sv.router, sv.strategy, pr.adapter.c_str(), pr.prefix.data(), static_cast<int>(pr.prefix.size()),
                              sv.mean_load_pct, 30ll * 1000 * 1000, addr, sizeof(addr), &ep_token);
    if (rc) {
      release_all();
      sv.errors_total.fetch_add(1);
      return send_error(w, 504, "request timeout while finding host");
    }
    tokens_held.push_back(ep_token);
    const int replica = atoi(addr + 4);  // "gpu:<i>"
    b200_engine* eng = sv.replicas[replica];
    b200_sampling sp{};
    sp.max_tokens = max_tokens;
    sp.temperature = static_cast<float>(pr.temperature);
    sp.top_p = static_cast<float>(pr.top_p);
    sp.top_k = pr.top_k;
    sp.has_seed = pr.has_seed ? 1 : 0;
    sp.seed = static_cast<uint64_t>(pr.seed);
    sp.ignore_eos = pr.ignore_eos ? 1 : 0;
    sp.logprobs = pr.logprobs >= 0 ? 1 : 0;
    sp.top_logprobs = std::max(pr.logprobs, 0);
    sp.presence_penalty = static_cast<float>(pr.presence);
    sp.frequency_penalty = static_cast<float>(pr.frequency);
    sp.repetition_penalty = static_cast<float>(pr.repetition);
    sp.min_p = static_cast<float>(pr.min_p);
    sp.min_tokens = pr.min_tokens;
    sp.num_logit_bias = static_cast<int>(pr.bias_ids.size());
    sp.logit_bias_ids = pr.bias_ids.empty() ? nullptr : pr.bias_ids.data();
    sp.logit_bias_values = pr.bias_values.empty() ? nullptr : pr.bias_values.data();
    sp.prompt_logprobs = plp_n >= 0 ? 1 : 0;
    sp.top_prompt_logprobs = std::max(plp_n, 0);
    std::vector<int32_t> stops = pr.stop_ids;
    if (sv.real_tok && !pr.ignore_eos) {   // the checkpoint's end-of-turn / end-of-text tokens end the generation
      for (const char* name : {"<|eot_id|>", "<|end_of_text|>"}) {
        const int32_t t = b200_tokenizer_token_id(sv.real_tok, name);
        if (t >= 0) stops.push_back(t);
      }
    }
    sp.num_stop_ids = static_cast<int>(stops.size());
    sp.stop_ids = stops.empty() ? nullptr : stops.data();
    // one element per choice (vLLM's n): its request id, output ids and logprob records, detokeniser and text_offset
    struct Choice {
      uint64_t rid = 0;
      std::vector<int32_t> all;
      std::vector<LpRecord> all_lp;
      DetokStream detok;
      size_t text_off = 0;   // completions stream: text_offset runs across chunks
      bool echoed = false;
      int fin = 0;
      b200_usage usage{};
    };
    std::vector<Choice> ch(static_cast<size_t>(pr.n));
    std::vector<uint64_t> rids(ch.size());
    bool failed = false;
    if (sv.faults[replica]->load() < 0) failed = true;  // permanent fault: stands for an engine in the failed state
    else if (sv.faults[replica]->load() > 0 && sv.faults[replica]->fetch_sub(1) > 0) failed = true;
    if (!failed && b200_submit_n(eng, ids.data(), static_cast<int>(ids.size()), &sp, pr.n, rids.data())) failed = true;

    std::vector<LpRecord> prompt_lp;   // the prompt records (plp_n >= 0), read with the first token; every choice shares them
    bool have_plp = false;
    // an echo's leading records: the first prompt token's null entry, then the prompt records
    auto echo_recs = [&] {
      std::vector<LpRecord> e{LpRecord{ids[0], 0.f, {}}};
      e[0].none = true;
      e.insert(e.end(), prompt_lp.begin(), prompt_lp.end());
      return e;
    };
    const bool want_lp = pr.logprobs >= 0;
    // a token's string in logprobs: the single-id lossy decode (vLLM's tokenizer.decode([id])), or the synthetic piece
    auto token_str = [&](int32_t id) { return sv.real_tok ? tokenizer_token_text(sv.real_tok, id) : sv.tok.piece(id); };
    for (size_t c = 0; c < ch.size(); ++c) {
      ch[c].rid = rids[c];
      ch[c].detok.tok = sv.real_tok;
    }
    bool sent_any = false;
    if (!failed) {
      int32_t buf[256];
      std::vector<float> lpv, top_lp;
      std::vector<int32_t> top_ids;
      if (want_lp) {
        lpv.resize(256);
        top_lp.resize(256 * B200_MAX_LOGPROBS);
        top_ids.resize(256 * B200_MAX_LOGPROBS);
      }
      std::vector<uint64_t> live;
      for (;;) {
        live.clear();
        for (auto& c : ch)
          if (!c.fin) live.push_back(c.rid);
        if (live.empty()) break;
        b200_wait_any(eng, live.data(), static_cast<int>(live.size()), 200000);
        // the choices in ascending index: within one engine step their chunks go out in that order
        for (size_t ci = 0; ci < ch.size() && !failed; ++ci) {
          Choice& c = ch[ci];
          if (c.fin) continue;
          int n = 0;
          const int prc = want_lp ? b200_poll_logprobs(eng, c.rid, buf, lpv.data(), top_ids.data(), top_lp.data(), 256, &n, &c.fin, &c.usage)
                                  : b200_poll(eng, c.rid, buf, 256, &n, &c.fin, &c.usage);
          if (prc) { failed = true; break; }
          if (c.fin == B200_FINISH_ERROR && !sent_any) { failed = true; break; }
          if (plp_n >= 0 && !have_plp && n > 0) {   // published no later than the first token
            const int np = static_cast<int>(ids.size()) - 1;
            std::vector<float> plv(std::max(np, 1)), ptl(static_cast<size_t>(std::max(np, 1)) * B200_MAX_LOGPROBS);
            std::vector<int32_t> prk(std::max(np, 1)), pti(static_cast<size_t>(std::max(np, 1)) * B200_MAX_LOGPROBS);
            int got = 0;
            if (b200_poll_prompt_logprobs(eng, c.rid, plv.data(), prk.data(), pti.data(), ptl.data(), np, &got) || got != np) { failed = true; break; }
            for (int k = 0; k < np; ++k) {
              LpRecord r{ids[k + 1], plv[k], {}};
              r.rank = prk[k];
              for (int j = 0; j < plp_n; ++j)
                r.top.emplace_back(pti[static_cast<size_t>(k) * B200_MAX_LOGPROBS + j], ptl[static_cast<size_t>(k) * B200_MAX_LOGPROBS + j]);
              prompt_lp.push_back(std::move(r));
            }
            have_plp = true;
          }
          std::vector<LpRecord> recs;
          for (int i = 0; want_lp && i < n; ++i) {
            LpRecord r{buf[i], lpv[i], {}};
            for (int j = 0; j < pr.logprobs; ++j)
              r.top.emplace_back(top_ids[static_cast<size_t>(i) * B200_MAX_LOGPROBS + j], top_lp[static_cast<size_t>(i) * B200_MAX_LOGPROBS + j]);
            recs.push_back(std::move(r));
          }
          const std::string index = "{\"index\":" + std::to_string(ci);
          if (pr.stream && n > 0) {
            if (!sent_any) {
              w.begin(200, "text/event-stream; charset=utf-8");
              // chat: one role chunk per choice first (vLLM's chat_completion/serving.py)
              for (size_t k = 0; pr.chat && k < ch.size(); ++k)
                w.write("data: " + head + ",\"choices\":[{\"index\":" + std::to_string(k) +
                        ",\"delta\":{\"role\":\"assistant\",\"content\":\"\"},\"logprobs\":null,\"finish_reason\":null}]}\n\n");
              sent_any = true;
            }
            for (int i = 0; i < n; ++i) {
              const bool last = c.fin && i == n - 1;
              const std::string fr = last ? std::string("\"") + finish_str(c.fin) + "\"" : "null";
              // one chunk per token; with a real tokenizer a chunk carries the text that token completed (possibly none: a
              // token may end inside a UTF-8 sequence), and the last chunk also what was still held
              const std::string text = sv.real_tok ? c.detok.push(buf[i]) + (last ? c.detok.flush() : std::string()) : sv.tok.piece(buf[i]);
              std::string piece = json_str(text);
              std::string lpj = "null";
              if (want_lp && pr.chat) lpj = "{\"content\":[" + chat_lp_content(recs[i], token_str) + "]}";
              else if (want_lp) lpj = completion_lp({recs[i]}, c.text_off, token_str, pr.logprobs);
              if (pr.echo && !c.echoed) {
                // vLLM's first echo chunk: the prompt and its records, then the first token's unless max_tokens was 0.  The
                // offsets of later chunks count the generated text only, as in vLLM.
                piece = json_str(echo_text + (echo_only ? std::string() : text));
                if (want_lp) {
                  std::vector<LpRecord> e = echo_recs();
                  if (!echo_only) e.push_back(recs[i]);
                  lpj = completion_lp(e, 0, token_str, pr.logprobs);
                }
                c.echoed = true;
              }
              c.text_off += utf8_len(text);
              if (pr.chat)
                w.write("data: " + head + ",\"choices\":[" + index + ",\"delta\":{\"content\":" + piece + "},\"logprobs\":" + lpj + ",\"finish_reason\":" + fr +
                        (last ? ",\"stop_reason\":null" : "") + "}]}\n\n");
              else
                w.write("data: " + head + ",\"choices\":[" + index + ",\"text\":" + piece + ",\"logprobs\":" + lpj + ",\"finish_reason\":" + fr + ",\"stop_reason\":null}],\"usage\":null}\n\n");
            }
          }
          c.all.insert(c.all.end(), buf, buf + n);
          c.all_lp.insert(c.all_lp.end(), recs.begin(), recs.end());
        }
        if (failed) break;
        if (w.gone) {  // client disconnected: abort every choice and free its KV blocks
          for (auto& c : ch) b200_abort(eng, c.rid);
          break;
        }
      }
      for (auto& c : ch) b200_release(eng, c.rid);
    }
    if (failed) {
      if (b200_engine_is_failed(eng) || sv.faults[replica]->load() < 0) sv.drop_replica(replica);
      if (attempt < sv.max_retries) {
        sv.retries_total.fetch_add(1);
        continue;
      }
      release_all();
      sv.errors_total.fetch_add(1);
      return send_error(w, 502, "proxy: exceeded retries");
    }
    release_all();
    if (w.gone) return 499;
    // usage: the prompt once, the completion tokens of every choice
    b200_usage usage = ch[0].usage;
    for (size_t c = 1; c < ch.size(); ++c) usage.completion_tokens += ch[c].usage.completion_tokens;
    if (pr.stream) {
      if (!sent_any) w.begin(200, "text/event-stream; charset=utf-8");
      if (pr.include_usage) w.write("data: " + head + ",\"choices\":[],\"usage\":" + usage_json(usage) + "}\n\n");
      w.write("data: [DONE]\n\n");
    } else {
      // vLLM's prompt_logprobs: on every completions choice, once at the top level of a chat response
      const std::string plj = plp_n >= 0 ? ",\"prompt_logprobs\":" + prompt_lp_json(prompt_lp, token_str) : std::string();
      std::string out = "{\"id\":\"" + id + "\",\"object\":\"" + (pr.chat ? "chat.completion" : "text_completion") +
                        "\",\"created\":" + std::to_string(created) + ",\"model\":" + json_str(pr.requested_model) + ",\"choices\":[";
      for (size_t ci = 0; ci < ch.size(); ++ci) {
        const Choice& c = ch[ci];
        std::string text;
        if (sv.real_tok) {
          DetokStream whole;
          whole.tok = sv.real_tok;
          for (auto t : c.all) text += whole.push(t);
          text += whole.flush();
        } else {
          for (auto t : c.all) text += sv.tok.piece(t);
        }
        out += (ci ? ",{\"index\":" : "{\"index\":") + std::to_string(ci) + ",";
        if (pr.echo) text = echo_text + (echo_only ? std::string() : text);
        if (pr.chat) out += "\"message\":{\"role\":\"assistant\",\"content\":" + json_str(text) + "},";
        else out += "\"text\":" + json_str(text) + ",";
        std::string lpj = "null";
        if (want_lp && pr.chat) {
          lpj = "{\"content\":[";
          for (size_t k = 0; k < c.all_lp.size(); ++k) lpj += (k ? "," : "") + chat_lp_content(c.all_lp[k], token_str);
          lpj += "]}";
        } else if (want_lp && pr.echo) {
          std::vector<LpRecord> e = echo_recs();
          if (!echo_only) e.insert(e.end(), c.all_lp.begin(), c.all_lp.end());
          lpj = completion_lp(e, 0, token_str, pr.logprobs);
        } else if (want_lp) {
          lpj = completion_lp(c.all_lp, 0, token_str, pr.logprobs);
        }
        out += "\"logprobs\":" + lpj + ",\"finish_reason\":\"" + finish_str(c.fin) + "\",\"stop_reason\":null" + (pr.chat ? "" : plj) + "}";
      }
      out += "],\"usage\":" + usage_json(usage) + (pr.chat ? plj : "") + "}";
      w.begin(200, "application/json");
      w.write(out);
    }
    return 200;
  }
}

// Standard base64 with padding (RFC 4648 §4), as Python's base64.b64encode gives.
static std::string base64(const uint8_t* p, size_t n) {
  static const char* a = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
  std::string o;
  o.reserve((n + 2) / 3 * 4);
  for (size_t i = 0; i < n; i += 3) {
    const uint32_t v = (static_cast<uint32_t>(p[i]) << 16) | (i + 1 < n ? static_cast<uint32_t>(p[i + 1]) << 8 : 0) |
                       (i + 2 < n ? p[i + 2] : 0);
    o += a[(v >> 18) & 63];
    o += a[(v >> 12) & 63];
    o += i + 1 < n ? a[(v >> 6) & 63] : '=';
    o += i + 2 < n ? a[v & 63] : '=';
  }
  return o;
}

// The embedding inputs and options of a /v1/embeddings body (vLLM 0.22's EmbeddingCompletionRequest).  Returns 0 or 400
// with *err set.  Every field the engine does not implement is refused, never dropped.
struct EmbedRequest {
  std::vector<std::vector<int32_t>> inputs;
  bool base64 = false;
  bool normalize = true;
};
static int parse_embed_body(const Server& sv, const char* body, size_t len, EmbedRequest* er, std::string* err) {
  JVal root;
  std::string jerr;
  if (!JParser(body, len).parse(&root, &jerr) || root.type != JVal::Obj) { *err = "bad request: expected a JSON object"; return 400; }
  auto bad = [&](const std::string& m) { *err = "bad request: " + m; return 400; };
  auto present = [&](const char* k) { const JVal* v = root.get(k); return v && v->type != JVal::Null; };
  if (present("dimensions"))
    return bad("Model \"" + sv.model + "\" does not support matryoshka representation, changing output dimensions will lead to poor results.");
  if (const JVal* v = root.get("embed_dtype"); v && v->type != JVal::Null && !(v->type == JVal::Str && v->str == "float32"))
    return bad("embed_dtype other than float32 is not supported by this engine");
  if (const JVal* v = root.get("endianness"); v && v->type != JVal::Null &&
      !(v->type == JVal::Str && (v->str == "native" || v->str == "little")))
    return bad("endianness other than native or little is not supported by this engine");
  if (present("truncate_prompt_tokens")) return bad("truncate_prompt_tokens is not supported by this engine");
  if (present("messages")) return bad("chat-form embeddings (messages) are not supported by this engine");
  if (const JVal* v = root.get("encoding_format"); v && v->type != JVal::Null) {
    if (v->type == JVal::Str && v->str == "base64") er->base64 = true;
    else if (!(v->type == JVal::Str && v->str == "float")) return bad("encoding_format must be \"float\" or \"base64\"");
  }
  if (const JVal* v = root.get("use_activation"); v && v->type != JVal::Null) {
    if (v->type != JVal::Bool) return bad("use_activation must be a boolean or null");
    er->normalize = v->b;
  }
  bool special = true;
  if (const JVal* v = root.get("add_special_tokens"); v && v->type != JVal::Null) {
    if (v->type != JVal::Bool) return bad("add_special_tokens must be a boolean");
    special = v->b;
  }
  auto text_ids = [&](const std::string& s, std::vector<int32_t>* ids) {
    if (sv.real_tok) {
      if (special && tokenizer_bos(sv.real_tok) >= 0) ids->push_back(tokenizer_bos(sv.real_tok));
      std::vector<int32_t> buf(s.size() + 16);
      int64_t n = b200_tokenizer_encode(sv.real_tok, s.data(), s.size(), 1, buf.data(), buf.size());
      if (n > static_cast<int64_t>(buf.size())) {
        buf.resize(static_cast<size_t>(n));
        n = b200_tokenizer_encode(sv.real_tok, s.data(), s.size(), 1, buf.data(), buf.size());
      }
      if (n > 0) ids->insert(ids->end(), buf.begin(), buf.begin() + n);
    } else {
      sv.tok.encode(s, ids);
    }
  };
  auto id_list = [&](const JVal& a, std::vector<int32_t>* ids) {
    for (auto& e : a.arr) {
      if (e.type != JVal::Num || e.num != std::floor(e.num) || !(e.num >= 0 && e.num < sv.tok.vocab)) return false;
      ids->push_back(static_cast<int32_t>(e.num));
    }
    return true;
  };
  const JVal* in = root.get("input");
  if (!in || in->type == JVal::Null) return bad("input is required");
  const std::string shape = "input must be a string, a list of strings, a list of token ids or a list of token id lists";
  if (in->type == JVal::Str) {
    er->inputs.emplace_back();
    text_ids(in->str, &er->inputs.back());
  } else if (in->type == JVal::Arr) {
    if (in->arr.empty()) return bad("input must not be empty");
    const JVal::Type t0 = in->arr[0].type;
    for (auto& e : in->arr)
      if (e.type != t0) return bad(shape);
    if (t0 == JVal::Num) {
      er->inputs.emplace_back();
      if (!id_list(*in, &er->inputs.back())) return bad("token ids must be integers in [0, " + std::to_string(sv.tok.vocab) + ")");
    } else if (t0 == JVal::Str) {
      for (auto& e : in->arr) {
        er->inputs.emplace_back();
        text_ids(e.str, &er->inputs.back());
      }
    } else if (t0 == JVal::Arr) {
      for (auto& e : in->arr) {
        er->inputs.emplace_back();
        if (!id_list(e, &er->inputs.back())) return bad("token ids must be integers in [0, " + std::to_string(sv.tok.vocab) + ")");
      }
    } else {
      return bad(shape);
    }
  } else {
    return bad(shape);
  }
  for (auto& ids : er->inputs) {
    if (ids.empty()) return bad("input must not be empty");
    // vLLM 0.22 renderers/params.py _token_len_check, with the 0 output tokens of a pooling request; it says "at least"
    // when the count is max_model_len + 1, the length its tokenizer truncates a longer text to
    if (static_cast<int>(ids.size()) > sv.max_model_len) {
      const std::string n = (static_cast<int>(ids.size()) == sv.max_model_len + 1 ? "at least " : "") + std::to_string(ids.size());
      return bad("This model's maximum context length is " + std::to_string(sv.max_model_len) +
                 " tokens. However, you requested 0 output tokens and your prompt contains " + n +
                 " input tokens, for a total of " + n + " tokens. Please reduce the length of the input prompt or the number "
                 "of requested output tokens.");
    }
  }
  return 0;
}

// /v1/embeddings on a pooling server: every input is one engine request, all submitted before any is waited on; the
// response is vLLM's EmbeddingResponse with data in input order.  Retries follow serve_inference.  The response is one
// write at the end, and the writer reports a client that went away only when a write fails: as for a non-streaming
// completion, such a client is noticed at that write (status 499), after its requests finished and were released.
static int serve_embeddings(Server& sv, const std::string& path, const std::string& ctype, const char* body, size_t len,
                            Writer& w) {
  ParsedRequest pr;
  std::string err;
  if (int st = parse_request(sv, path, ctype, body, len, &pr, &err)) return send_error(w, st, err);
  EmbedRequest er;
  if (int st = parse_embed_body(sv, body, len, &er, &err)) return send_error(w, st, err);
  {
    std::lock_guard<std::mutex> lk(sv.mmu);
    ++sv.active[pr.requested_model];
  }
  sv.requests_total.fetch_add(1);
  struct Dec {
    Server& s;
    std::string m;
    ~Dec() {
      std::lock_guard<std::mutex> lk(s.mmu);
      --s.active[m];
    }
  } dec{sv, pr.requested_model};
  const size_t n_in = er.inputs.size();
  std::vector<uint64_t> tokens_held;
  auto release_all = [&] {
    for (auto t : tokens_held) b200_router_done(sv.router, t);
    tokens_held.clear();
  };
  for (int attempt = 0;; ++attempt) {
    char addr[64];
    uint64_t ep_token = 0;
    if (b200_router_pick(sv.router, sv.strategy, pr.adapter.c_str(), "", 0, sv.mean_load_pct, 30ll * 1000 * 1000, addr,
                         sizeof(addr), &ep_token)) {
      release_all();
      sv.errors_total.fetch_add(1);
      return send_error(w, 504, "request timeout while finding host");
    }
    tokens_held.push_back(ep_token);
    const int replica = atoi(addr + 4);  // "gpu:<i>"
    b200_engine* eng = sv.replicas[replica];
    bool failed = false;
    if (sv.faults[replica]->load() < 0) failed = true;
    else if (sv.faults[replica]->load() > 0 && sv.faults[replica]->fetch_sub(1) > 0) failed = true;
    std::vector<uint64_t> rids;
    for (size_t i = 0; i < n_in && !failed; ++i) {
      uint64_t rid = 0;
      if (b200_submit_embed(eng, er.inputs[i].data(), static_cast<int>(er.inputs[i].size()), er.normalize ? 1 : 0, &rid)) failed = true;
      else rids.push_back(rid);
    }
    std::vector<float> vecs(n_in * static_cast<size_t>(sv.hidden));
    std::vector<b200_usage> usage(n_in);
    std::vector<int> fin(n_in, 0);
    for (size_t i = 0; i < rids.size() && !failed;) {
      if (fin[i]) { ++i; continue; }
      b200_wait(eng, rids[i], 200000);
      if (b200_poll_embedding(eng, rids[i], vecs.data() + i * sv.hidden, sv.hidden, &fin[i], &usage[i])) failed = true;
      else if (fin[i] && fin[i] != B200_FINISH_STOP) failed = true;
    }
    for (auto r : rids) b200_release(eng, r);   // releasing an unfinished request (a failed attempt) aborts it
    if (failed) {
      if (b200_engine_is_failed(eng) || sv.faults[replica]->load() < 0) sv.drop_replica(replica);
      if (attempt < sv.max_retries) {
        sv.retries_total.fetch_add(1);
        continue;
      }
      release_all();
      sv.errors_total.fetch_add(1);
      return send_error(w, 502, "proxy: exceeded retries");
    }
    release_all();
    int prompt_tokens = 0;
    for (auto& u : usage) prompt_tokens += u.prompt_tokens;
    std::string out = "{\"id\":\"embd-" + hex_id(32) + "\",\"object\":\"list\",\"created\":" +
                      std::to_string(static_cast<long>(time(nullptr))) + ",\"model\":" + json_str(pr.requested_model) + ",\"data\":[";
    char num[32];
    for (size_t i = 0; i < n_in; ++i) {
      out += (i ? ",{\"index\":" : "{\"index\":") + std::to_string(i) + ",\"object\":\"embedding\",\"embedding\":";
      const float* v = vecs.data() + i * sv.hidden;
      if (er.base64) {
        // the little-endian fp32 bytes (vLLM's float32 embed_dtype at native endianness on x86 / aarch64)
        out += "\"" + base64(reinterpret_cast<const uint8_t*>(v), static_cast<size_t>(sv.hidden) * sizeof(float)) + "\"";
      } else {
        out += "[";
        for (int k = 0; k < sv.hidden; ++k) {
          snprintf(num, sizeof(num), "%.9g", static_cast<double>(v[k]));   // 9 significant digits round-trip an fp32
          out += (k ? "," : "");
          out += num;
        }
        out += "]";
      }
      out += "}";
    }
    out += "],\"usage\":{\"prompt_tokens\":" + std::to_string(prompt_tokens) + ",\"total_tokens\":" + std::to_string(prompt_tokens) +
           ",\"completion_tokens\":0,\"prompt_tokens_details\":null}}";
    w.begin(200, "application/json");
    w.write(out);
    return w.gone ? 499 : 200;
  }
}

// The pairs and options of a /v1/rerank body (vLLM 0.22's RerankRequest; its types were checked by parse_request).  Returns
// 0 or 400 with *err set.  Every field the engine does not implement is refused, never dropped.
struct RerankRequest {
  std::vector<std::string> documents;
  std::vector<std::vector<int32_t>> pairs;   // the tokenized (query, document i)
  int top_n = 0;
  bool use_activation = true;
};
static int parse_rerank_body(const Server& sv, const char* body, size_t len, RerankRequest* rr, std::string* err) {
  JVal root;
  std::string jerr;
  if (!JParser(body, len).parse(&root, &jerr) || root.type != JVal::Obj) { *err = "bad request: expected a JSON object"; return 400; }
  auto bad = [&](const std::string& m) { *err = "bad request: " + m; return 400; };
  auto present = [&](const char* k) { const JVal* v = root.get(k); return v && v->type != JVal::Null; };
  for (const char* k : {"max_tokens_per_query", "max_tokens_per_doc"})
    if (const JVal* v = root.get(k); v && v->type != JVal::Null && !(v->type == JVal::Num && v->num == 0))
      return bad(std::string(k) + " (per-document truncation) is not supported by this engine");
  for (const char* k : {"truncate_prompt_tokens", "instruction", "chat_template_kwargs", "priority"})
    if (present(k)) return bad(std::string(k) + " is not supported by this engine");
  if (sv.num_labels != 1)   // vLLM's ScoringOutput.from_base: a rerank score is the one logit of its row
    return bad("pooled_data should be a scalar score: /v1/rerank needs a score head of 1 label, this model has " +
               std::to_string(sv.num_labels));
  if (const JVal* v = root.get("use_activation"); v && v->type != JVal::Null) {
    if (v->type != JVal::Bool) return bad("use_activation must be a boolean or null");
    rr->use_activation = v->b;
  }
  bool special = true;
  if (const JVal* v = root.get("add_special_tokens"); v && v->type != JVal::Null) {
    if (v->type != JVal::Bool) return bad("add_special_tokens must be a boolean");
    special = v->b;
  }
  if (const JVal* v = root.get("top_n"); v && v->type == JVal::Num)
    rr->top_n = v->num > 2147483647.0 ? 2147483647 : v->num < -2147483648.0 ? -2147483647 - 1 : static_cast<int>(v->num);
  std::string query;
  if (const JVal* v = root.get("query"); v && v->type == JVal::Str) query = v->str;
  if (const JVal* v = root.get("documents"); v && v->type == JVal::Arr)
    for (auto& d : v->arr) rr->documents.push_back(d.type == JVal::Str ? d.str : "");
  if (rr->documents.empty()) return bad("documents must not be empty");
  for (auto& d : rr->documents) {
    rr->pairs.emplace_back();
    std::vector<int32_t>& ids = rr->pairs.back();
    if (sv.real_tok) {
      tokenizer_encode_pair(sv.real_tok, query, d, sv.join_pair, special, &ids);
    } else {   // the synthetic tokenizer has no special tokens: the two encodings, concatenated
      sv.tok.encode(sv.join_pair ? query + d : query, &ids);
      if (!sv.join_pair) sv.tok.encode(d, &ids);
    }
    if (ids.empty()) return bad("the query and document must not both be empty");
    // the embeddings route's message: vLLM 0.22 renderers/params.py _token_len_check with 0 output tokens
    if (static_cast<int>(ids.size()) > sv.max_model_len) {
      const std::string n = (static_cast<int>(ids.size()) == sv.max_model_len + 1 ? "at least " : "") + std::to_string(ids.size());
      return bad("This model's maximum context length is " + std::to_string(sv.max_model_len) +
                 " tokens. However, you requested 0 output tokens and your prompt contains " + n +
                 " input tokens, for a total of " + n + " tokens. Please reduce the length of the input prompt or the number "
                 "of requested output tokens.");
    }
  }
  return 0;
}

// The shortest decimal that reads back as the same double (Python's float repr, which vLLM's JSON dump of a score
// prints); the double holds the fp32 score exactly, so a client recovers the score to the bit.
static std::string shortest_double(double v) {
  char b[40];
  for (int p = 1; p <= 17; ++p) {
    snprintf(b, sizeof(b), "%.*g", p, v);
    if (strtod(b, nullptr) == v) break;
  }
  return b;
}

// /v1/rerank on a score-head server: every (query, document) pair is one engine request, all submitted before any is
// waited on; the response is vLLM's RerankResponse, results sorted by score (descending, stable: equal scores keep the
// document order, as Python's sort(reverse=True) does) and cut to top_n when 0 < top_n < len(documents).  Retries and
// the 499 of a client that went away follow serve_embeddings.
static int serve_rerank(Server& sv, const std::string& path, const std::string& ctype, const char* body, size_t len,
                        Writer& w) {
  ParsedRequest pr;
  std::string err;
  if (int st = parse_request(sv, path, ctype, body, len, &pr, &err)) return send_error(w, st, err);
  RerankRequest rr;
  if (int st = parse_rerank_body(sv, body, len, &rr, &err)) return send_error(w, st, err);
  {
    std::lock_guard<std::mutex> lk(sv.mmu);
    ++sv.active[pr.requested_model];
  }
  sv.requests_total.fetch_add(1);
  struct Dec {
    Server& s;
    std::string m;
    ~Dec() {
      std::lock_guard<std::mutex> lk(s.mmu);
      --s.active[m];
    }
  } dec{sv, pr.requested_model};
  const size_t n_in = rr.pairs.size();
  std::vector<uint64_t> tokens_held;
  auto release_all = [&] {
    for (auto t : tokens_held) b200_router_done(sv.router, t);
    tokens_held.clear();
  };
  for (int attempt = 0;; ++attempt) {
    char addr[64];
    uint64_t ep_token = 0;
    if (b200_router_pick(sv.router, sv.strategy, pr.adapter.c_str(), "", 0, sv.mean_load_pct, 30ll * 1000 * 1000, addr,
                         sizeof(addr), &ep_token)) {
      release_all();
      sv.errors_total.fetch_add(1);
      return send_error(w, 504, "request timeout while finding host");
    }
    tokens_held.push_back(ep_token);
    const int replica = atoi(addr + 4);  // "gpu:<i>"
    b200_engine* eng = sv.replicas[replica];
    bool failed = false;
    if (sv.faults[replica]->load() < 0) failed = true;
    else if (sv.faults[replica]->load() > 0 && sv.faults[replica]->fetch_sub(1) > 0) failed = true;
    std::vector<uint64_t> rids;
    for (size_t i = 0; i < n_in && !failed; ++i) {
      uint64_t rid = 0;
      if (b200_submit_score(eng, rr.pairs[i].data(), static_cast<int>(rr.pairs[i].size()), rr.use_activation ? 1 : 0, &rid)) failed = true;
      else rids.push_back(rid);
    }
    std::vector<float> scores(n_in);
    std::vector<b200_usage> usage(n_in);
    std::vector<int> fin(n_in, 0);
    for (size_t i = 0; i < rids.size() && !failed;) {
      if (fin[i]) { ++i; continue; }
      b200_wait(eng, rids[i], 200000);
      if (b200_poll_score(eng, rids[i], &scores[i], 1, &fin[i], &usage[i])) failed = true;
      else if (fin[i] && fin[i] != B200_FINISH_STOP) failed = true;
    }
    for (auto r : rids) b200_release(eng, r);   // releasing an unfinished request (a failed attempt) aborts it
    if (failed) {
      if (b200_engine_is_failed(eng) || sv.faults[replica]->load() < 0) sv.drop_replica(replica);
      if (attempt < sv.max_retries) {
        sv.retries_total.fetch_add(1);
        continue;
      }
      release_all();
      sv.errors_total.fetch_add(1);
      return send_error(w, 502, "proxy: exceeded retries");
    }
    release_all();
    int prompt_tokens = 0;
    for (auto& u : usage) prompt_tokens += u.prompt_tokens;
    std::vector<size_t> order(n_in);
    for (size_t i = 0; i < n_in; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return scores[a] > scores[b]; });
    if (rr.top_n > 0 && static_cast<size_t>(rr.top_n) < n_in) order.resize(static_cast<size_t>(rr.top_n));
    std::string out = "{\"id\":\"score-" + hex_id(32) + "\",\"model\":" + json_str(pr.requested_model) +
                      ",\"usage\":{\"prompt_tokens\":" + std::to_string(prompt_tokens) + ",\"total_tokens\":" +
                      std::to_string(prompt_tokens) + "},\"results\":[";
    for (size_t k = 0; k < order.size(); ++k) {
      const size_t i = order[k];
      out += (k ? ",{\"index\":" : "{\"index\":") + std::to_string(i) + ",\"document\":{\"text\":" + json_str(rr.documents[i]) +
             ",\"multi_modal\":null},\"relevance_score\":" + shortest_double(static_cast<double>(scores[i])) + "}";
    }
    out += "]}";
    w.begin(200, "application/json");
    w.write(out);
    return w.gone ? 499 : 200;
  }
}

static std::string metrics_text(Server& sv) {
  std::string o;
  o += "# HELP kubeai_inference_requests_active The number of active requests by model\n# TYPE kubeai_inference_requests_active gauge\n";
  {
    std::lock_guard<std::mutex> lk(sv.mmu);
    for (auto& kv : sv.active)
      o += "kubeai_inference_requests_active{request_model=" + json_str(kv.first) + ",request_type=\"http\"} " + std::to_string(kv.second) + "\n";
  }
  {
    const int64_t n = b200_router_metrics(sv.router, nullptr, 0);
    if (n > 0) {
      std::string rm(static_cast<size_t>(n) + 1, '\0');
      b200_router_metrics(sv.router, &rm[0], rm.size());
      rm.resize(static_cast<size_t>(n));
      o += rm;
    }
  }
  o += "# TYPE b200_requests_total counter\nb200_requests_total " + std::to_string(sv.requests_total.load()) + "\n";
  o += "# TYPE b200_request_retries_total counter\nb200_request_retries_total " + std::to_string(sv.retries_total.load()) + "\n";
  for (size_t i = 0; i < sv.replicas.size(); ++i) {
    b200_stats st;
    if (b200_stats_get(sv.replicas[i], &st)) continue;
    char b[1024];
    snprintf(b, sizeof(b),
             "b200_engine_steps_total{replica=\"%zu\"} %lld\nb200_engine_running{replica=\"%zu\"} %d\nb200_engine_waiting{replica=\"%zu\"} %d\n"
             "b200_engine_kv_blocks_free{replica=\"%zu\"} %lld\nb200_engine_kv_blocks_total{replica=\"%zu\"} %lld\n"
             "b200_engine_prompt_tokens_total{replica=\"%zu\"} %lld\nb200_engine_cached_prompt_tokens_total{replica=\"%zu\"} %lld\n"
             "b200_engine_generated_tokens_total{replica=\"%zu\"} %lld\nb200_engine_preemptions_total{replica=\"%zu\"} %lld\n"
             "b200_engine_last_step_device_us{replica=\"%zu\"} %.1f\n",
             i, (long long)st.steps, i, st.running, i, st.waiting, i, (long long)st.kv_blocks_free, i, (long long)st.kv_blocks_total, i,
             (long long)st.prompt_tokens, i, (long long)st.cached_prompt_tokens, i, (long long)st.generated_tokens, i,
             (long long)st.preemptions, i, st.last_step_device_us);
    o += b;
    // speculative decoding, vLLM's counters vllm:spec_decode_num_drafts, vllm:spec_decode_num_draft_tokens,
    // vllm:spec_decode_num_accepted_tokens and vllm:spec_decode_num_accepted_tokens_per_pos{position} (zero when off)
    snprintf(b, sizeof(b),
             "b200_engine_spec_decode_num_drafts_total{replica=\"%zu\"} %lld\n"
             "b200_engine_spec_decode_num_draft_tokens_total{replica=\"%zu\"} %lld\n"
             "b200_engine_spec_decode_num_accepted_tokens_total{replica=\"%zu\"} %lld\n",
             i, (long long)st.spec_drafts, i, (long long)st.spec_draft_tokens, i, (long long)st.spec_accepted_tokens);
    o += b;
    for (int j = 0; j < B200_MAX_SPEC_TOKENS; ++j) {
      snprintf(b, sizeof(b), "b200_engine_spec_decode_num_accepted_tokens_per_pos_total{replica=\"%zu\",position=\"%d\"} %lld\n", i, j,
               (long long)st.spec_accepted_per_pos[j]);
      o += b;
    }
  }
  return o;
}

// openaiserver.NewHandler route table (handler.go:20-49) + /metrics + /healthz.
static int handle(Server& sv, const std::string& method, const std::string& full_path, const std::string& ctype,
                  const char* body, size_t len, Writer& w) {
  std::string path = full_path.substr(0, full_path.find('?'));
  if (path == "/healthz" || path == "/readyz") {
    w.begin(200, "text/plain");
    w.write("ok\n");
    return 200;
  }
  if (path == "/metrics") {
    w.begin(200, "text/plain; version=0.0.4");
    w.write(metrics_text(sv));
    return 200;
  }
  if (path.rfind("/openai/", 0) != 0) {
    w.begin(404, "text/plain");
    w.write("404 page not found\n");
    return 404;
  }
  path = path.substr(7);  // http.StripPrefix("/openai", ...)
  if (path == "/v1/models" && method == "GET") {
    // openaiserver/models.go:13-77 (static: one model + adapters)
    const std::string feat = sv.num_labels > 0 ? "Reranking" : sv.pooling ? "TextEmbedding" : "TextGeneration";
    std::string o = "{\"object\":\"list\",\"data\":[{\"id\":" + json_str(sv.model) + ",\"object\":\"model\",\"created\":0,\"owned_by\":\"kubeai-b200\",\"features\":[\"" + feat + "\"]}";
    for (auto& a : sv.adapters)
      o += ",{\"id\":" + json_str(sv.model + "_" + a) + ",\"object\":\"model\",\"created\":0,\"owned_by\":\"kubeai-b200\",\"features\":[\"" + feat + "\"]}";
    o += "]}";
    w.begin(200, "application/json");
    w.write(o);
    return 200;
  }
  // "X-Proxy: lingo" (handler.go:60) is added by the HTTP layer below / by the Go shim
  if (sv.num_labels > 0) {
    if (path == "/v1/rerank") return serve_rerank(sv, path, ctype, body, len, w);
    if (path == "/v1/chat/completions" || path == "/v1/completions" || path == "/v1/embeddings" || path == "/v1/audio/transcriptions")
      return send_error(w, 404, "model not found: this engine serves Reranking only");
  }
  if (sv.pooling && sv.num_labels == 0) {
    if (path == "/v1/embeddings") return serve_embeddings(sv, path, ctype, body, len, w);
    if (path == "/v1/chat/completions" || path == "/v1/completions" || path == "/v1/rerank" || path == "/v1/audio/transcriptions")
      return send_error(w, 404, "model not found: this engine serves TextEmbedding only");
  }
  if (path == "/v1/chat/completions" || path == "/v1/completions") return serve_inference(sv, path, ctype, body, len, w);
  if (path == "/v1/embeddings" || path == "/v1/rerank" || path == "/v1/audio/transcriptions")
    return send_error(w, 404, "model not found: this engine serves TextGeneration only");
  w.begin(404, "text/plain");
  w.write("404 page not found\n");
  return 404;
}

// ------------------------------------------------------------------ minimal HTTP/1.1 front (thread per connection)
namespace {

struct ConnWriter {
  int fd;
  bool chunked = false;
  bool head_sent = false;
  bool failed = false;
  static bool send_all(int fd, const char* p, size_t n) {
    while (n) {
      ssize_t k = ::send(fd, p, n, MSG_NOSIGNAL);
      if (k <= 0) {
        if (k < 0 && errno == EINTR) continue;
        return false;
      }
      p += k;
      n -= static_cast<size_t>(k);
    }
    return true;
  }
};

int conn_begin(void* ud, int status, const char* ctype) {
  ConnWriter* c = static_cast<ConnWriter*>(ud);
  if (status == 0) return 0;
  static const std::map<int, const char*> text = {{200, "OK"}, {400, "Bad Request"}, {404, "Not Found"}, {499, "Client Closed Request"},
                                                  {500, "Internal Server Error"}, {502, "Bad Gateway"}, {504, "Gateway Timeout"}};
  auto it = text.find(status);
  char h[512];
  c->chunked = true;
  int n = snprintf(h, sizeof(h), "HTTP/1.1 %d %s\r\nContent-Type: %s\r\nX-Proxy: lingo\r\nCache-Control: no-cache\r\nTransfer-Encoding: chunked\r\nConnection: keep-alive\r\n\r\n",
                   status, it == text.end() ? "Status" : it->second, ctype);
  c->head_sent = true;
  if (!ConnWriter::send_all(c->fd, h, static_cast<size_t>(n))) c->failed = true;
  return c->failed ? 1 : 0;
}

int conn_write(void* ud, const char* data, size_t len) {
  ConnWriter* c = static_cast<ConnWriter*>(ud);
  if (c->failed || len == 0) return c->failed ? 1 : 0;
  char h[32];
  int n = snprintf(h, sizeof(h), "%zx\r\n", len);
  std::string frame(h, static_cast<size_t>(n));
  frame.append(data, len);
  frame += "\r\n";
  if (!ConnWriter::send_all(c->fd, frame.data(), frame.size())) c->failed = true;
  return c->failed ? 1 : 0;
}

void serve_conn(Server* sv, int fd) {
  int one = 1;
  setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
  timeval tv{Server::kIdleTimeoutS, 0};
  setsockopt(fd, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof(tv));
  setsockopt(fd, SOL_SOCKET, SO_SNDTIMEO, &tv, sizeof(tv));
  std::string buf;
  char tmp[16384];
  for (;;) {
    // read headers
    size_t hend;
    while ((hend = buf.find("\r\n\r\n")) == std::string::npos) {
      ssize_t k = ::recv(fd, tmp, sizeof(tmp), 0);
      if (k <= 0) goto done;
      buf.append(tmp, static_cast<size_t>(k));
      if (buf.size() > (1 << 20)) goto done;
    }
    {
      std::string headers = buf.substr(0, hend);
      size_t body_off = hend + 4;
      size_t le = headers.find("\r\n");
      std::string reqline = headers.substr(0, le);
      std::string method = reqline.substr(0, reqline.find(' '));
      size_t p1 = reqline.find(' '), p2 = reqline.rfind(' ');
      std::string path = p1 != std::string::npos && p2 > p1 ? reqline.substr(p1 + 1, p2 - p1 - 1) : "/";
      size_t clen = 0;
      std::string ctype;
      bool close_after = false;
      size_t pos = le == std::string::npos ? headers.size() : le + 2;
      while (pos < headers.size()) {
        size_t e = headers.find("\r\n", pos);
        if (e == std::string::npos) e = headers.size();
        std::string line = headers.substr(pos, e - pos);
        pos = e + 2;
        size_t c = line.find(':');
        if (c == std::string::npos) continue;
        std::string k = line.substr(0, c), v = line.substr(c + 1);
        while (!v.empty() && v.front() == ' ') v.erase(v.begin());
        for (auto& ch : k) ch = static_cast<char>(tolower(ch));
        if (k == "content-length") clen = static_cast<size_t>(strtoull(v.c_str(), nullptr, 10));
        else if (k == "content-type") ctype = v;
        else if (k == "connection") { for (auto& ch : v) ch = static_cast<char>(tolower(ch)); close_after = v == "close"; }
      }
      if (clen > (64u << 20)) goto done;
      while (buf.size() < body_off + clen) {
        ssize_t k = ::recv(fd, tmp, sizeof(tmp), 0);
        if (k <= 0) goto done;
        buf.append(tmp, static_cast<size_t>(k));
      }
      ConnWriter cw{fd};
      b200_response_writer rw{&cw, conn_begin, conn_write};
      Writer w{&rw};
      handle(*sv, method, path, ctype, buf.data() + body_off, clen, w);
      if (cw.head_sent && !cw.failed) ConnWriter::send_all(fd, "0\r\n\r\n", 5);
      buf.erase(0, body_off + clen);
      if (cw.failed || close_after || sv->stopping) goto done;
    }
  }
done:
  {
    std::lock_guard<std::mutex> lk(sv->conn_mu);
    sv->conn_fds.erase(fd);
  }
  close(fd);
  sv->live_conns.fetch_sub(1);  // last touch of *sv: the destructor waits for this count to reach zero
}

}  // namespace
}  // namespace b200

using namespace b200;

struct b200_server {
  Server impl;
};

extern "C" {

int b200_server_create(const b200_server_config* cfg, b200_engine* const* replicas, int32_t n, b200_server** out) {
  if (!cfg || !replicas || n <= 0 || !out || !cfg->model) { set_error("b200_server_create: bad arguments"); return B200_ERR_INVALID; }
  b200_server* s = new (std::nothrow) b200_server();
  if (!s) { set_error("host OOM"); return B200_ERR_OOM; }
  Server& sv = s->impl;
  sv.model = cfg->model;
  if (cfg->adapters) {
    std::string a(cfg->adapters);
    size_t p = 0;
    while (p <= a.size()) {
      size_t q = a.find(',', p);
      if (q == std::string::npos) q = a.size();
      if (q > p) sv.adapters.insert(a.substr(p, q - p));
      p = q + 1;
    }
  }
  sv.strategy = cfg->strategy;
  // api/k8s/v1/model_types.go:173-209 defaults
  sv.mean_load_pct = cfg->mean_load_pct > 0 ? cfg->mean_load_pct : 125;
  sv.replication = cfg->replication > 0 ? cfg->replication : 256;
  sv.prefix_chars = cfg->prefix_char_length > 0 ? cfg->prefix_char_length : 100;
  sv.max_retries = cfg->max_retries >= 0 ? cfg->max_retries : 3;
  sv.default_max_tokens = cfg->default_max_tokens > 0 ? cfg->default_max_tokens : 256;
  sv.tok.vocab = cfg->vocab > 258 ? cfg->vocab : 128256;
  sv.max_model_len = cfg->max_model_len > 0 ? cfg->max_model_len : 2048;
  sv.sampling = cfg->enable_sampling != 0;
  sv.logprobs = cfg->enable_logprobs != 0;
  sv.edits = cfg->enable_logits_processors != 0;
  sv.prompt_lp = cfg->enable_prompt_logprobs != 0;
  sv.max_n = cfg->max_n;
  // the replicas share one runner: a server serves generation or embeddings, never both
  for (int i = 0, seen = 0; i < n; ++i) {
    if (!replicas[i]) continue;
    const bool pool = engine_runner(replicas[i]) == B200_RUNNER_POOLING;
    if (seen && pool != sv.pooling) {
      delete s;
      set_error("b200_server_create: the replicas mix the generate and pooling runners");
      return B200_ERR_INVALID;
    }
    // a server serves embeddings or one score head, never both
    if (seen && (engine_num_labels(replicas[i]) != sv.num_labels || (engine_score_join_pair(replicas[i]) != 0) != sv.join_pair)) {
      set_error("b200_server_create: the replicas mix heads (num_labels %d and %d)", sv.num_labels, engine_num_labels(replicas[i]));
      delete s;
      return B200_ERR_INVALID;
    }
    ++seen;
    sv.pooling = pool;
    sv.hidden = engine_hidden(replicas[i]);
    sv.num_labels = engine_num_labels(replicas[i]);
    sv.join_pair = engine_score_join_pair(replicas[i]) != 0;
  }
  if (b200_router_create(sv.replication, &sv.router)) { delete s; return B200_ERR_INVALID; }
  std::vector<std::string> names;
  std::string ad = cfg->adapters ? cfg->adapters : "";
  sv.adapters_csv = ad;
  sv.dead.assign(static_cast<size_t>(n), 0);
  for (int i = 0; i < n; ++i) {
    sv.replicas.push_back(replicas[i]);
    names.push_back("gpu-" + std::to_string(i));
    sv.addrs.push_back("gpu:" + std::to_string(i));
    sv.faults.emplace_back(new std::atomic<int>(0));
  }
  std::vector<const char*> np, ap, dp;
  for (int i = 0; i < n; ++i) { np.push_back(names[i].c_str()); ap.push_back(sv.addrs[i].c_str()); dp.push_back(ad.c_str()); }
  if (int rc = b200_router_set_endpoints(sv.router, np.data(), ap.data(), dp.data(), n)) { delete s; return rc; }
  *out = s;
  return 0;
}

void b200_server_destroy(b200_server* s) { delete s; }

int b200_server_handle(b200_server* s, const char* method, const char* path, const char* content_type, const char* body,
                       size_t body_len, const b200_response_writer* writer) {
  if (!s || !method || !path || !writer) { set_error("b200_server_handle: bad arguments"); return B200_ERR_INVALID; }
  Writer w{writer};
  return handle(s->impl, method, path, content_type ? content_type : "", body ? body : "", body ? body_len : 0, w);
}

/* apiutils.ParseRequest on its own (for parity tests against internal/apiutils/request_test.go and the Prefix tables):
 * returns 0 or the HTTP status of the error; out_json gets {"model","adapter","requested_model","prefix"} or {"error"}. */
int b200_server_parse_request(b200_server* s, const char* path, const char* content_type, const char* body, size_t body_len,
                              int32_t prefix_chars, char* out_json, size_t cap) {
  if (!s || !path || !out_json || cap == 0) { set_error("b200_server_parse_request: bad arguments"); return B200_ERR_INVALID; }
  Server& sv = s->impl;
  ParsedRequest pr;
  std::string err;
  const int saved = sv.prefix_chars;
  if (prefix_chars >= 0) sv.prefix_chars = prefix_chars;
  std::string p(path);
  if (p.rfind("/openai", 0) == 0) p = p.substr(7);
  const int st = parse_request(sv, p, content_type ? content_type : "", body ? body : "", body ? body_len : 0, &pr, &err);
  sv.prefix_chars = saved;
  std::string o = st ? "{\"error\":" + json_str(err) + "}"
                     : "{\"model\":" + json_str(pr.model) + ",\"adapter\":" + json_str(pr.adapter) + ",\"requested_model\":" +
                           json_str(pr.requested_model) + ",\"prefix\":" + json_str(pr.prefix) + "}";
  snprintf(out_json, cap, "%s", o.c_str());
  return st;
}

int b200_server_listen(b200_server* s, const char* host, int32_t port, int32_t* bound_port) {
  if (!s) { set_error("null server"); return B200_ERR_INVALID; }
  Server& sv = s->impl;
  int fd = socket(AF_INET, SOCK_STREAM, 0);
  if (fd < 0) { set_error("socket: %s", strerror(errno)); return B200_ERR_INVALID; }
  int one = 1;
  setsockopt(fd, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
  sockaddr_in a{};
  a.sin_family = AF_INET;
  a.sin_port = htons(static_cast<uint16_t>(port));
  inet_pton(AF_INET, host && *host ? host : "127.0.0.1", &a.sin_addr);
  if (bind(fd, reinterpret_cast<sockaddr*>(&a), sizeof(a)) || listen(fd, 1024)) {
    set_error("bind/listen: %s", strerror(errno));
    close(fd);
    return B200_ERR_INVALID;
  }
  socklen_t al = sizeof(a);
  getsockname(fd, reinterpret_cast<sockaddr*>(&a), &al);
  if (bound_port) *bound_port = ntohs(a.sin_port);
  sv.listen_fd = fd;
  sv.acceptor = std::thread([&sv, fd] {
    while (!sv.stopping) {
      int c = accept(fd, nullptr, nullptr);
      if (c < 0) {
        if (sv.stopping) break;
        if (errno == EINTR) continue;
        break;
      }
      if (sv.live_conns.load() >= Server::kMaxConns) {
        static const char busy[] = "HTTP/1.1 503 Service Unavailable\r\nContent-Length: 0\r\nConnection: close\r\n\r\n";
        (void)!::send(c, busy, sizeof(busy) - 1, MSG_NOSIGNAL);
        close(c);
        continue;
      }
      {
        std::lock_guard<std::mutex> lk(sv.conn_mu);
        if (sv.stopping) { close(c); break; }
        sv.conn_fds.insert(c);
      }
      sv.live_conns.fetch_add(1);
      std::thread(serve_conn, &sv, c).detach();
    }
  });
  return 0;
}

int b200_speculative_config_parse(const char* json, b200_config* cfg) {
  if (!json || !cfg) { set_error("b200_speculative_config_parse: bad arguments"); return B200_ERR_INVALID; }
  JVal v;
  std::string err;
  JParser jp(json, strlen(json));
  if (!jp.parse(&v, &err)) { set_error("speculative-config: %s", err.c_str()); return B200_ERR_INVALID; }
  if (v.type != JVal::Obj) { set_error("speculative-config: expected a JSON object"); return B200_ERR_INVALID; }
  int k = 0, mn = 0, mx = 0;
  bool has_method = false;
  for (auto& kv : v.obj) {
    const JVal& x = kv.second;
    if (kv.first == "method") {
      if (x.type != JVal::Str || x.str != "ngram") {
        set_error("speculative-config: only \"method\": \"ngram\" is supported (got %s)", x.type == JVal::Str ? x.str.c_str() : "a non-string");
        return B200_ERR_INVALID;
      }
      has_method = true;
    } else if (kv.first == "num_speculative_tokens" || kv.first == "prompt_lookup_min" || kv.first == "prompt_lookup_max") {
      const bool lookup = kv.first != "num_speculative_tokens";
      if (lookup && x.is_null()) continue;   // unset
      if (x.type != JVal::Num || !x.is_int || x.num < 1 || x.num > 1e6) {
        set_error("speculative-config: %s must be an integer >= 1", kv.first.c_str());
        return B200_ERR_INVALID;
      }
      (kv.first == "num_speculative_tokens" ? k : kv.first == "prompt_lookup_min" ? mn : mx) = static_cast<int>(x.num);
    } else {
      set_error("speculative-config: unsupported key \"%s\" (the ngram method takes num_speculative_tokens, "
                "prompt_lookup_min and prompt_lookup_max)", kv.first.c_str());
      return B200_ERR_INVALID;
    }
  }
  if (!has_method) { set_error("speculative-config: \"method\" is required (only \"ngram\" is supported)"); return B200_ERR_INVALID; }
  if (k < 1 || k > B200_MAX_SPEC_TOKENS) {
    set_error("speculative-config: num_speculative_tokens must be in 1..%d for the ngram method, got %d", B200_MAX_SPEC_TOKENS, k);
    return B200_ERR_INVALID;
  }
  if (mn && mx && mn > mx) {
    set_error("speculative-config: prompt_lookup_min=%d must be <= prompt_lookup_max=%d", mn, mx);
    return B200_ERR_INVALID;
  }
  cfg->num_speculative_tokens = k;
  cfg->prompt_lookup_min = mn;
  cfg->prompt_lookup_max = mx;
  return 0;
}

int b200_server_metrics(b200_server* s, char* buf, size_t cap) {
  if (!s || !buf || cap == 0) { set_error("bad arguments"); return B200_ERR_INVALID; }
  std::string m = metrics_text(s->impl);
  snprintf(buf, cap, "%s", m.c_str());
  return static_cast<int>(m.size());
}

int b200_server_set_tokenizer(b200_server* s, const b200_tokenizer* t) {
  if (!s) { set_error("b200_server_set_tokenizer: bad arguments"); return B200_ERR_INVALID; }
  if (t && b200_tokenizer_vocab_size(t) > s->impl.tok.vocab) {
    set_error("the tokenizer has %d ids, the model's vocabulary %d", b200_tokenizer_vocab_size(t), s->impl.tok.vocab);
    return B200_ERR_INVALID;
  }
  s->impl.real_tok = t;
  return 0;
}

int64_t b200_server_render_prompt(b200_server* s, const char* path, const char* content_type, const char* body, size_t len, int32_t* ids,
                                  size_t cap) {
  if (!s || !path || (!body && len)) { set_error("b200_server_render_prompt: bad arguments"); return -1; }
  ParsedRequest pr;
  std::string err;
  if (int st = parse_request(s->impl, path, content_type ? content_type : "application/json", body, len, &pr, &err)) {
    set_error("%d %s", st, err.c_str());
    return -1;
  }
  std::vector<int32_t> out;
  render_prompt(s->impl, pr, &out);
  for (size_t i = 0; i < out.size() && i < cap; ++i) ids[i] = out[i];
  return static_cast<int64_t>(out.size());
}

int b200_server_inject_fault(b200_server* s, int32_t replica, int32_t count) {
  if (!s || replica < 0 || replica >= static_cast<int>(s->impl.replicas.size())) { set_error("bad replica"); return B200_ERR_INVALID; }
  s->impl.faults[replica]->store(count);
  return 0;
}

int b200_tokenize(int32_t vocab, const char* text, size_t len, int32_t* out, int32_t cap) {
  Tokenizer t;
  t.vocab = vocab;
  std::vector<int32_t> ids;
  t.encode(std::string(text ? text : "", text ? len : 0), &ids);
  const int n = static_cast<int>(ids.size());
  if (out) memcpy(out, ids.data(), static_cast<size_t>(std::min(n, cap)) * 4);
  return n;
}

int b200_detokenize(int32_t vocab, const int32_t* ids, int32_t n, char* out, size_t cap) {
  Tokenizer t;
  t.vocab = vocab;
  std::string s;
  for (int i = 0; i < n; ++i) s += t.piece(ids[i]);
  if (out && cap) snprintf(out, cap, "%s", s.c_str());
  return static_cast<int>(s.size());
}

}  // extern "C"
