// Host text side of CT-Transformer punctuation (punc_text.cpp; no CUDA): the word split, the vocabulary lookup and the mini-sentence
// walk of CTTransformer.inference, run in lockstep over many texts.  Shared by fa_punc_walk_host (any scorer) and fa_punc_infer (the
// GPU forward as the scorer) in offline_punc.cu: there is one walk.
#pragma once
#include <stdint.h>
#include <functional>
#include <string>
#include <unordered_map>
#include <vector>

namespace fa_punc {

struct Vocab {
  std::unordered_map<std::string, int32_t> token_id;
  int32_t unk = -1;                                  // the id of "<unk>" (CharTokenizer's unk_symbol)
  std::vector<std::string> punc;                     // punc_list
  int32_t sentence_end_id = 3;
  int32_t split_size = 20;
  bool init(const std::vector<std::string>& tokens, const std::vector<std::string>& punc_list, int32_t sentence_end, int32_t split,
            std::string& err);
};

struct Result {
  std::vector<std::string> text;
  std::vector<std::vector<int32_t>> ids;             // punc_array per text, after the forced end
  int64_t steps = 0;                                 // lockstep scorer calls
};

// One lockstep step: ids [batch, t_max] row-major, row b valid for its first lens[b] entries (the rest 0) -> punc_out [batch, t_max]
// (only the valid entries are read).  Returns false and sets err on failure.
using Scorer = std::function<bool(const int32_t* ids, const int32_t* lens, int32_t batch, int32_t t_max, int32_t* punc_out, std::string& err)>;

// split_words of ct_transformer/utils.py:75-92: the text split at Python whitespace, ASCII runs one word, every other code point a word
std::vector<std::string> split_words(const std::string& text);

// CTTransformer.inference (ct_transformer/model.py:309-473) for every text at once: step s scores window s of every text that still has
// one as one batch.  max_window > 0: a window with more words fails the call before the step's scorer runs, naming the text.
bool walk(const Vocab& v, const char* const* texts, int32_t n, int64_t max_window, const Scorer& score, Result& out, std::string& err);

}  // namespace fa_punc
