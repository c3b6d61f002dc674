// C++ side of the BPE tokenizer (tokenizer.cc) for the serving shell: incremental detokenisation of a token stream.
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

struct b200_tokenizer;

namespace b200 {

// raw bytes one token id stands for (byte-level symbols mapped back; added tokens: their content, nothing for a special one
// when skip_special)
void tokenizer_token_bytes(const b200_tokenizer* t, int32_t id, bool skip_special, std::string* out);
// ids of the Llama-3 control tokens (-1 if the vocabulary lacks one)
int32_t tokenizer_bos(const b200_tokenizer* t);
int32_t tokenizer_eot(const b200_tokenizer* t);
// a cross-encoder's (query a, document b) ids, as vLLM tokenizes a score pair: join false = HF tokenizer(text=a,
// text_pair=b) through the tokenizer.json's pair template (use_sep_token = true), join true = tokenizer(text=a + b)
// through its single template (use_sep_token = false).  special false (add_special_tokens = false), or a tokenizer.json
// without a TemplateProcessing post-processor: the encodings are concatenated without special tokens.
void tokenizer_encode_pair(const b200_tokenizer* t, const std::string& a, const std::string& b, bool join, bool special,
                           std::vector<int32_t>* out);
// one id decoded on its own, special tokens kept, invalid UTF-8 replaced by U+FFFD (HF tokenizer.decode([id]))
std::string tokenizer_token_text(const b200_tokenizer* t, int32_t id);

// A token may end in the middle of a UTF-8 sequence (byte-level BPE): push() returns only text that is complete, holding an
// unfinished tail until the next token completes it; bytes that can never become valid are replaced by U+FFFD, as a lossy
// decode of the whole sequence would.  Concatenating every push() and the final flush() equals decoding all ids at once.
struct DetokStream {
  const b200_tokenizer* tok = nullptr;
  bool skip_special = true;
  std::string pending;
  std::string push(int32_t id);
  std::string flush();
};

}  // namespace b200
