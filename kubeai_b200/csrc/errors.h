// Thread-local error string shared by all C-ABI translation units.
#pragma once

namespace b200 {
void set_error(const char* fmt, ...);
int require_device();            // B200_ERR_NO_DEVICE (+message) when no GPU is present
int cuda_fail(const char* what, int rc);
}  // namespace b200
struct b200_engine;
namespace b200 {
// The gate_up weight named `name` was just filled in logical order ([gate rows | up rows]) through its device pointer:
// move it to the engine's physical layout (64-row gate/up blocks interleaved).  Used by the checkpoint loader.
int engine_relayout_gate_up(b200_engine* e, const char* name);
// b200_config.runner and hidden size of an engine (the serving shell routes and sizes embeddings by them)
int engine_runner(const b200_engine* e);
int engine_hidden(const b200_engine* e);
// b200_config.num_labels (0 = no score head) and score_join_pair of an engine (the serving shell routes /v1/rerank and
// tokenizes its pairs by them)
int engine_num_labels(const b200_engine* e);
int engine_score_join_pair(const b200_engine* e);
}
