// Host text side of CT-Transformer punctuation (punc_text.cpp; no CUDA): the word split, the vocabulary lookup and the mini-sentence
// walk of CTTransformer.inference, run in lockstep over many texts.  walk() runs it over one call's texts; the punctuation pool in
// offline_punc.cu steps the texts of many calls with the same operations (admit, compose, apply): there is one walk.
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

// One text's walk: its words and token ids, the window the next step scores, the unfinished tail carried into it, the text and
// punctuation ids so far.  It depends on no other text, so texts of any number of calls can share a step.
struct Text {
  std::vector<std::string> words;
  std::vector<int32_t> ids;
  int64_t n_windows = 0, next = 0;                 // split_to_mini_sentence's window count; the window the next step scores
  std::vector<std::string> cache_words;            // the unfinished tail carried into the next window
  std::vector<int32_t> cache_ids;
  std::string text;
  std::vector<int32_t> punc;
  bool active() const { return next < n_windows; }
};

// The walk in three operations.  admit: the word split, the vocabulary lookup and the window count of one text (an empty or
// whitespace-only text has no window: "" and no ids).
Text admit(const Vocab& v, const char* text);
// the words of x's next window (the carried tail and up to split_size new words); false with the call's message when max_window > 0
// and they are more, `index` naming the text within its call
int64_t window_len(const Vocab& v, const Text& x);
bool check_window(const Vocab& v, const Text& x, int32_t index, int64_t max_window, std::string& err);
// One step over active texts: ids [batch, t_max], lens [batch] and a punc_out of the same shape for the scorer
struct Step {
  std::vector<int32_t> ids, lens, pout;
  int32_t batch = 0, t_max = 0;
};
void compose(const Vocab& v, const std::vector<Text*>& rows, Step& s);
// row b of a scored step into rows[b]: the tail carry, cache_pop_trigger_limit, capitalisation, the forced sentence end.  false with
// the message for an id outside the punctuation list.
bool apply(const Vocab& v, Text& x, const Step& s, int32_t b, std::string& err);

// CTTransformer.inference (ct_transformer/model.py:309-473) for every text at once: step s scores window s of every text that still has
// one as one batch.  max_window > 0: a window with more words fails the call before the step's scorer runs, naming the text.
bool walk(const Vocab& v, const char* const* texts, int32_t n, int64_t max_window, const Scorer& score, Result& out, std::string& err);

}  // namespace fa_punc
