// Load generator: the reference's benchmarks/multi-turn-chat-go restated in C++.
//   main.go:26-136            config, thread loading, seeded shuffle, trim to thread_count
//   benchmark/runner.go:153-187  Run: semaphore of max_concurrent_threads, one worker per thread
//   benchmark/runner.go:263-352  RunThread: one streaming chat completion per input message, history grows
//   benchmark/runner.go:189-250  summarizeResults: TTFT / ITL / throughput arithmetic
// Extensions the metric needs (BASELINE.json): p50/p99 TTFT (the Go Result only has means) and a
// synthetic thread generator with the published workload's shape (SURVEY.md §8d) because the
// ShareGPT file is not available offline.  Transports: in-process (b200_server_handle) or HTTP/1.1.
#include <arpa/inet.h>
#include <errno.h>
#include <math.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <sys/socket.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/b200engine.h"
#include "errors.h"
#include "hostutil.h"

namespace b200 {
namespace {

struct Msg {
  std::string role, content;
};
struct RequestResult {
  double duration = 0;
  std::vector<double> tt_chunks;
  int prompt_tokens = 0, cached_prompt_tokens = 0, completion_tokens = 0, total_tokens = 0;
};
struct HThread {
  std::vector<Msg> input, current;
  int requests = 0;
  std::vector<RequestResult> results;
  bool failed = false;
  std::string err;
};

struct SplitMix {
  uint64_t s;
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uniform() { return static_cast<double>(next() >> 11) * (1.0 / 9007199254740992.0); }
  double normal() {
    double u1 = uniform(), u2 = uniform();
    if (u1 < 1e-300) u1 = 1e-300;
    return sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
  }
};

// Incremental SSE consumer shared by both transports: feed bytes, it records chunk timings.
struct SseSink {
  RequestResult* rr;
  double t_chunk0;
  std::string buf, text, role;
  bool done = false, bad = false;
  std::string err;
  void feed(const char* d, size_t n) {
    buf.append(d, n);
    size_t pos;
    while ((pos = buf.find("\n\n")) != std::string::npos) {
      std::string ev = buf.substr(0, pos);
      buf.erase(0, pos + 2);
      if (ev.rfind("data: ", 0) != 0) continue;
      std::string payload = ev.substr(6);
      if (payload == "[DONE]") { done = true; continue; }
      JVal v;
      std::string e;
      if (!JParser(payload.data(), payload.size()).parse(&v, &e)) { bad = true; err = "stream: " + e; continue; }
      if (const JVal* er = v.get("error")) { bad = true; err = "stream: " + (er->type == JVal::Str ? er->str : std::string("error")); continue; }
      const JVal* ch = v.get("choices");
      // runner.go:319-328: a chunk counts iff len(Choices) > 0 && FinishReason in {"", null}
      if (ch && ch->type == JVal::Arr && !ch->arr.empty()) {
        const JVal* fr = ch->arr[0].get("finish_reason");
        if (!fr || fr->is_null() || (fr->type == JVal::Str && fr->str.empty())) {
          const double now = now_s();
          rr->tt_chunks.push_back(now - t_chunk0);
          if (const JVal* delta = ch->arr[0].get("delta")) {
            if (const JVal* c = delta->get("content"); c && c->type == JVal::Str) text += c->str;
            if (role.empty())
              if (const JVal* r = delta->get("role"); r && r->type == JVal::Str) role = r->str;
          }
        } else if (const JVal* delta = ch->arr[0].get("delta")) {
          // the finish_reason chunk still carries the last token's text (vLLM framing); the Go
          // client drops it from responseText as well as from the timings — mirrored here
          (void)delta;
        }
      }
      if (const JVal* u = v.get("usage"); u && u->type == JVal::Obj) {
        if (const JVal* x = u->get("prompt_tokens")) rr->prompt_tokens = static_cast<int>(x->num);
        if (const JVal* x = u->get("completion_tokens")) rr->completion_tokens = static_cast<int>(x->num);
        if (const JVal* x = u->get("total_tokens")) rr->total_tokens = static_cast<int>(x->num);
        if (const JVal* d = u->get("prompt_tokens_details"))
          if (const JVal* x = d->get("cached_tokens")) rr->cached_prompt_tokens = static_cast<int>(x->num);
      }
      t_chunk0 = now_s();  // runner.go:339
    }
  }
};

std::string request_body(const std::string& model, int max_tokens, float temperature, const std::vector<Msg>& msgs) {
  std::string b = "{\"model\":" + json_str(model) + ",\"messages\":[";
  for (size_t i = 0; i < msgs.size(); ++i) {
    if (i) b += ',';
    b += "{\"role\":" + json_str(msgs[i].role) + ",\"content\":" + json_str(msgs[i].content) + "}";
  }
  char t[64];
  snprintf(t, sizeof(t), "%g", temperature);
  b += "],\"max_tokens\":" + std::to_string(max_tokens) + ",\"stream\":true,\"temperature\":" + t +
       ",\"stream_options\":{\"include_usage\":true}}";
  return b;
}

struct Transport {
  b200_server* server = nullptr;  // in-process
  std::string host;
  int port = 0;
};

struct SinkCtx {
  SseSink* sink;
  int status = 0;
  std::string raw;
};
int sink_begin(void* ud, int status, const char*) {
  static_cast<SinkCtx*>(ud)->status = status;
  return 0;
}
int sink_write(void* ud, const char* d, size_t n) {
  SinkCtx* c = static_cast<SinkCtx*>(ud);
  if (c->status == 200) c->sink->feed(d, n);
  else c->raw.append(d, n);
  return 0;
}

bool do_request_inproc(Transport& tp, const std::string& body, SseSink* sink, std::string* err) {
  SinkCtx ctx{sink};
  b200_response_writer w{&ctx, sink_begin, sink_write};
  int st = b200_server_handle(tp.server, "POST", "/openai/v1/chat/completions", "application/json", body.data(), body.size(), &w);
  if (st != 200) {
    *err = "request: status " + std::to_string(st) + " " + ctx.raw;
    return false;
  }
  return true;
}

bool do_request_http(Transport& tp, const std::string& body, SseSink* sink, double timeout_s, std::string* err) {
  int fd = socket(AF_INET, SOCK_STREAM, 0);
  if (fd < 0) { *err = "socket"; return false; }
  sockaddr_in a{};
  a.sin_family = AF_INET;
  a.sin_port = htons(static_cast<uint16_t>(tp.port));
  inet_pton(AF_INET, tp.host.c_str(), &a.sin_addr);
  int one = 1;
  setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
  if (timeout_s > 0) {
    timeval tv{static_cast<long>(timeout_s), static_cast<long>((timeout_s - floor(timeout_s)) * 1e6)};
    setsockopt(fd, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof(tv));
  }
  if (connect(fd, reinterpret_cast<sockaddr*>(&a), sizeof(a))) { *err = std::string("connect: ") + strerror(errno); close(fd); return false; }
  std::string req = "POST /openai/v1/chat/completions HTTP/1.1\r\nHost: " + tp.host + "\r\nContent-Type: application/json\r\nAccept: text/event-stream\r\nConnection: close\r\nContent-Length: " +
                    std::to_string(body.size()) + "\r\n\r\n" + body;
  const char* p = req.data();
  size_t n = req.size();
  while (n) {
    ssize_t k = send(fd, p, n, MSG_NOSIGNAL);
    if (k <= 0) { *err = "send"; close(fd); return false; }
    p += k;
    n -= static_cast<size_t>(k);
  }
  std::string in;
  char tmp[8192];
  bool headers_done = false, chunked = false;
  int status = 0;
  std::string raw_body;
  size_t chunk_left = 0;
  bool ok = true;
  for (;;) {
    ssize_t k = recv(fd, tmp, sizeof(tmp), 0);
    if (k < 0) { *err = "recv timeout/error"; ok = false; break; }
    if (k == 0) break;
    in.append(tmp, static_cast<size_t>(k));
    if (!headers_done) {
      size_t he = in.find("\r\n\r\n");
      if (he == std::string::npos) continue;
      std::string h = in.substr(0, he);
      status = atoi(h.c_str() + 9);
      std::string hl = h;
      for (auto& c : hl) c = static_cast<char>(tolower(c));
      chunked = hl.find("transfer-encoding: chunked") != std::string::npos;
      in.erase(0, he + 4);
      headers_done = true;
    }
    // de-chunk
    while (!in.empty()) {
      if (!chunked) {
        if (status == 200) sink->feed(in.data(), in.size()); else raw_body += in;
        in.clear();
        break;
      }
      if (chunk_left == 0) {
        size_t le = in.find("\r\n");
        if (le == std::string::npos) break;
        chunk_left = strtoul(in.c_str(), nullptr, 16);
        in.erase(0, le + 2);
        if (chunk_left == 0) goto finished;
        chunk_left += 2;  // trailing CRLF
      }
      size_t take = std::min(chunk_left, in.size());
      size_t payload = chunk_left > 2 ? std::min(take, chunk_left - 2) : 0;
      if (payload) {
        if (status == 200) sink->feed(in.data(), payload); else raw_body.append(in.data(), payload);
      }
      in.erase(0, take);
      chunk_left -= take;
    }
    if (sink->done) break;
  }
finished:
  close(fd);
  if (ok && status != 200) { *err = "request: status " + std::to_string(status) + " " + raw_body; ok = false; }
  return ok;
}

// requests the running load generators of this process are about to have in flight (b200_harness_expected_inflight)
std::atomic<int64_t> g_expected_inflight{0};

// runner.go:263-352
void run_thread(Transport& tp, const b200_harness_config& cfg, HThread& t) {
  for (auto& m : t.input) {
    if (m.role == "user") break;
    t.current.push_back(m);
  }
  for (auto& m : t.input) {
    t.current.push_back(m);
    RequestResult rr;
    const double t0 = now_s();
    ++t.requests;
    SseSink sink{&rr, t0};
    std::string err;
    const std::string body = request_body(cfg.request_model, cfg.max_completion_tokens, cfg.temperature, t.current);
    bool ok = tp.server ? do_request_inproc(tp, body, &sink, &err) : do_request_http(tp, body, &sink, cfg.request_timeout_s, &err);
    if (ok && sink.bad) { ok = false; err = sink.err; }
    if (!ok) { t.failed = true; t.err = err; return; }
    t.current.push_back({sink.role, sink.text});
    rr.duration = now_s() - t0;
    t.results.push_back(std::move(rr));
  }
}

double percentile(std::vector<double>& v, double q) {
  if (v.empty()) return 0;
  std::sort(v.begin(), v.end());
  double idx = q * static_cast<double>(v.size() - 1);
  size_t lo = static_cast<size_t>(floor(idx)), hi = static_cast<size_t>(ceil(idx));
  return v[lo] + (v[hi] - v[lo]) * (idx - static_cast<double>(lo));
}

// Synthetic threads with the shape of the reference's large-exact.json (SURVEY.md §8d):
// 5..30 user messages per thread (clipped geometric, mean ~7.4), message length log-normal with
// mean ~50 tokens, total user content clipped to the prep script's 500..3000 characters
// (benchmarks/multi-turn-chat-go/Makefile:34-37, data/prepare-input-threads.py:49-58).
void synth_threads(const b200_harness_config& cfg, std::vector<HThread>* out) {
  SplitMix rng{static_cast<uint64_t>(cfg.seed) * 0x9E3779B97F4A7C15ull + 12345};
  Tokenizer tok;
  tok.vocab = cfg.vocab > 258 ? cfg.vocab : 128256;
  const double p = 1.0 / (cfg.synth_mean_msgs - 5.0 + 1.0);  // geometric on top of the minimum 5
  for (int i = 0; i < cfg.synth_threads; ++i) {
    HThread t;
    int n = 5;
    while (n < 30 && rng.uniform() > p) ++n;
    // per-message token counts, then rescale into the 500..3000 char window (5 chars per word)
    std::vector<int> words(n);
    int total = 0;
    const double mu = log(static_cast<double>(cfg.synth_mean_words)) - 0.5 * 0.6 * 0.6;
    for (int k = 0; k < n; ++k) {
      words[k] = std::max(2, static_cast<int>(exp(mu + 0.6 * rng.normal())));
      total += words[k];
    }
    const int lo = 100, hi = 600;  // 500..3000 chars / 5 chars per word
    if (total > hi || total < lo) {
      const double f = static_cast<double>(total > hi ? hi : lo) / static_cast<double>(total);
      for (auto& w : words) w = std::max(2, static_cast<int>(w * f));
    }
    for (int k = 0; k < n; ++k) {
      std::string s;
      for (int w = 0; w < words[k]; ++w) s += tok.piece(256 + static_cast<int>(rng.next() % static_cast<uint64_t>(tok.vocab - 258)));
      t.input.push_back({"user", s.substr(1)});  // drop the leading space of the first word
    }
    out->push_back(std::move(t));
  }
}

bool load_threads(const char* json, size_t len, std::vector<HThread>* out, std::string* err) {
  JVal root;
  if (!JParser(json, len).parse(&root, err) || root.type != JVal::Arr) {
    if (err->empty()) *err = "threads file must be a JSON array";
    return false;
  }
  for (auto& th : root.arr) {
    HThread t;
    if (const JVal* ms = th.get("messages"); ms && ms->type == JVal::Arr)
      for (auto& m : ms->arr) {
        const JVal* r = m.get("role");
        const JVal* c = m.get("content");
        t.input.push_back({r && r->type == JVal::Str ? r->str : "", c && c->type == JVal::Str ? c->str : ""});
      }
    out->push_back(std::move(t));
  }
  return true;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

void b200_harness_config_default(b200_harness_config* c) {
  memset(c, 0, sizeof(*c));
  c->request_model = "llama-3-8b";
  c->max_concurrent_threads = 128;
  c->max_completion_tokens = 40;   // runs/llama-3.1-8x-l4/run.ipynb cell 6
  c->temperature = 0.f;            // greedy (north star); sent explicitly
  c->thread_count = 0;
  c->seed = 2;
  c->request_timeout_s = 120.0;
  c->synth_threads = 1024;
  c->synth_mean_msgs = 7.38;
  c->synth_mean_words = 50;
  c->vocab = 128256;
}

int64_t b200_harness_expected_inflight(void) { return g_expected_inflight.load(); }

/* The synthetic thread list as JSON in the reference's input format (for sharding across ranks). */
int64_t b200_harness_synth_threads(const b200_harness_config* cfg, char* buf, size_t cap) {
  if (!cfg) { set_error("null config"); return B200_ERR_INVALID; }
  std::vector<HThread> threads;
  synth_threads(*cfg, &threads);
  std::string o = "[";
  for (size_t i = 0; i < threads.size(); ++i) {
    if (i) o += ',';
    o += "{\"id\":\"t" + std::to_string(i) + "\",\"messages\":[";
    for (size_t k = 0; k < threads[i].input.size(); ++k) {
      if (k) o += ',';
      o += "{\"role\":" + json_str(threads[i].input[k].role) + ",\"content\":" + json_str(threads[i].input[k].content) + "}";
    }
    o += "]}";
  }
  o += "]";
  if (buf && cap > o.size()) memcpy(buf, o.c_str(), o.size() + 1);
  return static_cast<int64_t>(o.size());
}

int b200_harness_run(b200_server* server, const char* host, int32_t port, const b200_harness_config* cfg,
                     const char* threads_json, size_t threads_len, b200_harness_result* out) {
  if (!cfg || !out || (!server && (!host || port <= 0))) { set_error("b200_harness_run: bad arguments"); return B200_ERR_INVALID; }
  if (cfg->max_concurrent_threads <= 0) { set_error("max_concurrent_threads (--max-concurrent-threads) must be greater than 0"); return B200_ERR_INVALID; }
  if (cfg->max_completion_tokens <= 0) { set_error("max_completion_tokens (--max-completion-tokens) must be greater than 0"); return B200_ERR_INVALID; }
  std::vector<HThread> threads;
  if (threads_json) {
    std::string err;
    if (!load_threads(threads_json, threads_len, &threads, &err)) { set_error("threads: %s", err.c_str()); return B200_ERR_INVALID; }
  } else {
    synth_threads(*cfg, &threads);
  }
  // main.go:98-116: seeded Fisher-Yates shuffle, then trim (Go's math/rand stream is not reproduced)
  {
    SplitMix rng{static_cast<uint64_t>(cfg->seed)};
    for (size_t i = threads.size(); i > 1; --i) std::swap(threads[i - 1], threads[rng.next() % i]);
    if (cfg->thread_count > 0 && static_cast<size_t>(cfg->thread_count) < threads.size()) threads.resize(static_cast<size_t>(cfg->thread_count));
  }
  Transport tp;
  tp.server = server;
  if (!server) { tp.host = host; tp.port = port; }

  // runner.go:153-187: semaphore + one worker per thread.  `expected` = conversations in progress + free slots that a
  // conversation still waiting to start will take: the requests this run is about to have in flight.  It changes only
  // when a conversation ends with none left to start, so a caller that steps the engine only while the engine holds
  // exactly that many unfinished requests sees the same batches on every run (b200_harness_expected_inflight).
  std::mutex mu;
  std::condition_variable cv;
  int slots = cfg->max_concurrent_threads;
  size_t not_started = threads.size();
  int64_t expected = static_cast<int64_t>(std::min<size_t>(static_cast<size_t>(slots), not_started));
  g_expected_inflight.fetch_add(expected);
  auto set_expected = [&](int64_t active) {   // under mu
    const int64_t e = active + static_cast<int64_t>(std::min<size_t>(static_cast<size_t>(slots), not_started));
    g_expected_inflight.fetch_add(e - expected);
    expected = e;
  };
  int64_t active = 0;
  std::vector<std::thread> workers;
  workers.reserve(threads.size());
  const double t0 = now_s();
  for (size_t i = 0; i < threads.size(); ++i) {
    {
      std::unique_lock<std::mutex> lk(mu);
      cv.wait(lk, [&] { return slots > 0; });
      --slots;
      --not_started;
      set_expected(++active);
    }
    workers.emplace_back([&, i] {
      run_thread(tp, *cfg, threads[i]);
      {
        std::lock_guard<std::mutex> lk(mu);
        ++slots;
        set_expected(--active);
      }
      cv.notify_one();
    });
  }
  for (auto& w : workers) w.join();
  g_expected_inflight.fetch_add(-expected);
  const double duration = now_s() - t0;

  // runner.go:189-250
  memset(out, 0, sizeof(*out));
  std::vector<double> ttfts, req_durs, itls;
  double total_itl_time = 0, total_itl_tokens = 0;
  long total_chunks = 0, total_input_msgs = 0;
  for (auto& t : threads) {
    out->request_count += t.requests;
    total_input_msgs += static_cast<long>(t.input.size());
    if (t.failed) { ++out->failed_threads; continue; }
    for (auto& rr : t.results) {
      int itl_chunks = 0;
      for (size_t c = 0; c < rr.tt_chunks.size(); ++c) {
        ++total_chunks;
        if (c == 0) ttfts.push_back(rr.tt_chunks[c]);
        else { total_itl_time += rr.tt_chunks[c]; itls.push_back(rr.tt_chunks[c]); ++itl_chunks; }
      }
      out->prompt_tokens += rr.prompt_tokens;
      out->cached_prompt_tokens += rr.cached_prompt_tokens;
      out->completion_tokens += rr.completion_tokens;
      out->total_tokens += rr.total_tokens;
      req_durs.push_back(rr.duration);
      total_itl_tokens += static_cast<double>(itl_chunks) / static_cast<double>(itl_chunks + 1) * rr.completion_tokens;
    }
  }
  auto mean = [](const std::vector<double>& v) { double s = 0; for (double x : v) s += x; return v.empty() ? 0.0 : s / static_cast<double>(v.size()); };
  out->duration_s = duration;
  out->input_thread_count = static_cast<int>(threads.size());
  out->input_messages_per_thread_mean = threads.empty() ? 0 : static_cast<double>(total_input_msgs) / static_cast<double>(threads.size());
  out->ttft_mean_s = mean(ttfts);
  out->itl_mean_s = total_itl_tokens > 0 ? total_itl_time / total_itl_tokens : 0;
  out->request_duration_mean_s = mean(req_durs);
  out->chunks_per_request_mean = out->request_count ? static_cast<double>(total_chunks) / out->request_count : 0;
  out->run_output_throughput = duration > 0 ? out->completion_tokens / duration : 0;
  out->run_total_throughput = duration > 0 ? out->total_tokens / duration : 0;
  out->ttft_p50_s = percentile(ttfts, 0.50);
  out->ttft_p90_s = percentile(ttfts, 0.90);
  out->ttft_p99_s = percentile(ttfts, 0.99);
  out->itl_p50_s = percentile(itls, 0.50);
  out->itl_p99_s = percentile(itls, 0.99);
  for (auto& t : threads)
    if (t.failed && out->first_error[0] == 0) snprintf(out->first_error, sizeof(out->first_error), "%s", t.err.c_str());
  return 0;
}

}  // extern "C"
