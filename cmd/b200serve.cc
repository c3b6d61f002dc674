// b200serve — the process entry a deployment runs: one engine per local GPU, the CHWBL / LeastLoad router over them,
// and the OpenAI-compatible HTTP front on :8000 under /openai/ — the three wiring lines of the reference's
// internal/manager/run.go:210,267-275 (loadbalancer.New, modelproxy.NewHandler, openaiserver.NewHandler) with the
// in-process engine in place of backend pods.  Everything else of cmd/main.go / manager.Run (K8s manager, autoscaler,
// messengers) is out of scope.
//
//   b200serve --gpus 8 --model llama-3-8b [--model-dir /models/llama-3-8b] [--strategy PrefixHash] [--port 8000]
//             [--speculative-config '{"method": "ngram", "num_speculative_tokens": 3, "prompt_lookup_max": 4}']
//             [--runner generate|pooling]   (default: pooling for a LlamaModel / MistralModel directory and for a
//                                            *ForSequenceClassification one, which serves /v1/rerank; else generate)
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <string>
#include <vector>

#include "../include/b200engine.h"

static volatile sig_atomic_t g_stop = 0;
static void on_signal(int) { g_stop = 1; }

int main(int argc, char** argv) {
  int gpus = 1, port = 8000, max_seqs = 128, max_len = 2048, budget = 2048;
  std::string model = "llama-3-8b", model_dir, strategy = "LeastLoad", host = "0.0.0.0", adapters, tokenizer_path;
  double kv_fraction = 0.85;
  unsigned long long seed = 0;
  bool greedy_only = false;
  std::string spec_json;   // vLLM's --speculative-config; speculation stays off without it
  std::string runner;      // vLLM's --runner: generate | pooling; default from the checkpoint's architecture
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    auto next = [&]() -> const char* { return i + 1 < argc ? argv[++i] : ""; };
    if (a == "--gpus") gpus = atoi(next());
    else if (a == "--port") port = atoi(next());
    else if (a == "--host") host = next();
    else if (a == "--model") model = next();
    else if (a == "--model-dir") model_dir = next();
    else if (a == "--adapters") adapters = next();
    else if (a == "--tokenizer") tokenizer_path = next();   // tokenizer.json; default: <model-dir>/tokenizer.json when present
    else if (a == "--strategy") strategy = next();
    else if (a == "--max-num-seqs") max_seqs = atoi(next());
    else if (a == "--max-model-len") max_len = atoi(next());
    else if (a == "--max-num-batched-tokens") budget = atoi(next());
    else if (a == "--gpu-memory-utilization") kv_fraction = atof(next());
    else if (a == "--seed") seed = strtoull(next(), nullptr, 10);
    else if (a == "--greedy-only") greedy_only = true;   // refuse temperature >= 1e-5 with a 400
    else if (a == "--speculative-config") spec_json = next();
    else if (a == "--runner") runner = next();
    else { fprintf(stderr, "unknown flag %s\n", a.c_str()); return 2; }
  }
  b200_config cfg;
  b200_config_default(&cfg);
  if (!model_dir.empty() && b200_config_from_hf(model_dir.c_str(), &cfg)) { fprintf(stderr, "config: %s\n", b200_last_error()); return 1; }
  cfg.max_num_seqs = max_seqs;
  cfg.max_model_len = max_len;
  cfg.max_batched_tokens = budget;
  cfg.kv_fraction = static_cast<float>(kv_fraction);
  cfg.seed = seed;
  if (runner == "generate") cfg.runner = B200_RUNNER_GENERATE;
  else if (runner == "pooling") cfg.runner = B200_RUNNER_POOLING;
  else if (!runner.empty()) { fprintf(stderr, "--runner must be generate or pooling, got %s\n", runner.c_str()); return 2; }
  if (!spec_json.empty() && b200_speculative_config_parse(spec_json.c_str(), &cfg)) { fprintf(stderr, "%s\n", b200_last_error()); return 2; }
  std::vector<b200_engine*> engines;
  for (int g = 0; g < gpus; ++g) {
    cfg.device = g;
    b200_engine* e = nullptr;
    if (b200_engine_create(&cfg, &e)) { fprintf(stderr, "engine %d: %s\n", g, b200_last_error()); return 1; }
    if (!model_dir.empty() && b200_engine_load_safetensors(e, model_dir.c_str())) { fprintf(stderr, "load: %s\n", b200_last_error()); return 1; }
    engines.push_back(e);
    fprintf(stderr, "[b200serve] replica gpu:%d ready\n", g);
  }
  b200_server_config sc;
  memset(&sc, 0, sizeof(sc));
  sc.model = model.c_str();
  sc.adapters = adapters.empty() ? nullptr : adapters.c_str();
  sc.strategy = strategy == "PrefixHash" ? B200_LB_PREFIX_HASH : B200_LB_LEAST_LOAD;
  sc.max_retries = 3;
  sc.vocab = cfg.vocab;
  sc.max_model_len = cfg.max_model_len;
  sc.enable_sampling = greedy_only ? 0 : 1;
  sc.enable_logprobs = 1;
  sc.enable_logits_processors = 1;
  sc.enable_prompt_logprobs = 1;
  sc.max_n = max_seqs;   // every choice of a request runs at once
  b200_server* srv = nullptr;
  if (b200_server_create(&sc, engines.data(), gpus, &srv)) { fprintf(stderr, "server: %s\n", b200_last_error()); return 1; }
  // the checkpoint's tokenizer + Llama-3 chat template when there is one; the synthetic tokenizer otherwise
  b200_tokenizer* tokenizer = nullptr;
  const bool explicit_tokenizer = !tokenizer_path.empty();
  if (tokenizer_path.empty() && !model_dir.empty()) {
    const std::string cand = model_dir + "/tokenizer.json";
    if (FILE* f = fopen(cand.c_str(), "rb")) { fclose(f); tokenizer_path = cand; }
  }
  if (!tokenizer_path.empty() && cfg.runner == B200_RUNNER_POOLING && !explicit_tokenizer &&
      b200_tokenizer_load(tokenizer_path.c_str(), &tokenizer)) {
    // an embedding checkpoint whose tokenizer is not of the Llama-3 pipeline is served through token-id inputs
    fprintf(stderr, "[b200serve] %s not loaded (%s): token-id inputs only\n", tokenizer_path.c_str(), b200_last_error());
    tokenizer_path.clear();
  }
  if (!tokenizer_path.empty()) {
    if ((!tokenizer && b200_tokenizer_load(tokenizer_path.c_str(), &tokenizer)) || b200_server_set_tokenizer(srv, tokenizer)) { fprintf(stderr, "tokenizer: %s\n", b200_last_error()); return 1; }
    fprintf(stderr, "[b200serve] tokenizer %s (%d ids)\n", tokenizer_path.c_str(), b200_tokenizer_vocab_size(tokenizer));
  }
  int bound = 0;
  if (b200_server_listen(srv, host.c_str(), port, &bound)) { fprintf(stderr, "listen: %s\n", b200_last_error()); return 1; }
  fprintf(stderr, "[b200serve] %s (%s) on http://%s:%d/openai/v1/chat/completions, %d replica(s)\n", model.c_str(), strategy.c_str(), host.c_str(), bound, gpus);
  signal(SIGINT, on_signal);
  signal(SIGTERM, on_signal);
  while (!g_stop) usleep(200000);
  b200_server_destroy(srv);
  if (tokenizer) b200_tokenizer_destroy(tokenizer);
  for (auto e : engines) b200_engine_destroy(e);
  return 0;
}
