/* Forced alignment through the plain C handle API: [start_ms, end_ms] for each token of a transcript (MonotonicAligner, fa-zh).
 * The transcript is tokenised as the fa-zh CharTokenizer does (split_with_space): stripped, split on single spaces, each piece looked
 * up in tokens.txt (one token per line), <unk> for a piece that is not there.
 * Model file: funasr_b200/pack.py write_aligner_model_file.
 * Build:  cc -std=c99 -Iinclude examples/offline_align_client.c -Lfunasr_b200 -lfunasr_b200 -o offline_align_client
 * usage:  offline_align_client <aligner.fab2> <tokens.txt> <audio.pcm (mono)> <transcript.txt> [sample_rate, default 16000]
 *                             [s16 | f32: the PCM's samples, default s16 (little endian; f32 in [-1, 1])]
 * Output: one "token start_ms end_ms" line per stamp. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "funasr_b200.h"

/* the whole file, NUL-terminated; NULL if it cannot be read */
static char* read_file(const char* path, long* bytes) {
  FILE* f = fopen(path, "rb");
  if (!f) return NULL;
  fseek(f, 0, SEEK_END);
  const long n = ftell(f);
  rewind(f);
  char* s = (char*)malloc(n > 0 ? (size_t)n + 1 : 1);
  const size_t got = s ? fread(s, 1, n > 0 ? (size_t)n : 0, f) : 0;
  fclose(f);
  if (!s) return NULL;
  s[got] = '\0';
  *bytes = (long)got;
  return s;
}

static int is_space(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\v' || c == '\f'; }

/* tokens.txt: one token per line, its id the line number; the tokens point into *text */
static char** read_tokens(const char* path, char** text, int32_t* n) {
  long bytes = 0;
  char* s = read_file(path, &bytes);
  if (!s) return NULL;
  int32_t cap = 1;
  for (long i = 0; i < bytes; ++i) cap += s[i] == '\n';
  char** tok = (char**)malloc(sizeof(char*) * (size_t)cap);
  *text = s;
  *n = 0;
  if (!tok) return NULL;
  char* line = s;
  for (long i = 0; i <= bytes; ++i) {
    if (i < bytes && s[i] != '\n') continue;
    if (i == bytes && line == s + bytes) break;            /* no line after the last newline */
    s[i] = '\0';
    if (i > 0 && s[i - 1] == '\r') s[i - 1] = '\0';
    tok[(*n)++] = line;
    line = s + i + 1;
  }
  return tok;
}

static int32_t lookup(char* const* tok, int32_t n, const char* piece) {
  for (int32_t i = 0; i < n; ++i)
    if (strcmp(tok[i], piece) == 0) return i;
  return -1;
}

int main(int argc, char** argv) {
  if (argc < 5) {
    fprintf(stderr, "usage: %s <aligner.fab2> <tokens.txt> <audio.pcm> <transcript.txt> [sample_rate] [s16|f32]\n", argv[0]);
    return 2;
  }
  const int32_t rate = argc > 5 ? atoi(argv[5]) : 16000;
  const int32_t f32 = argc > 6 && strcmp(argv[6], "f32") == 0;
  int32_t n_tok = 0;
  char* token_text = NULL;
  char** tok = read_tokens(argv[2], &token_text, &n_tok);
  const int32_t unk = tok ? lookup(tok, n_tok, "<unk>") : -1;
  if (!tok || unk < 0) {
    fprintf(stderr, "cannot read %s, or it has no <unk>\n", argv[2]);
    return 1;
  }
  long text_bytes = 0, pcm_bytes = 0;
  char* text = read_file(argv[4], &text_bytes);
  char* pcm = read_file(argv[3], &pcm_bytes);
  if (!text || !pcm) {
    fprintf(stderr, "cannot read %s or %s\n", argv[3], argv[4]);
    return 1;
  }
  /* str.strip().split(" "): every single space separates, so an empty transcript is one empty piece (<unk>), as in the tokenizer */
  char* b = text;
  char* e = text + text_bytes;
  while (b < e && is_space(*b)) ++b;
  while (e > b && is_space(e[-1])) --e;
  *e = '\0';
  int32_t n_ids = 1;
  for (char* p = b; *p; ++p) n_ids += *p == ' ';
  int32_t* ids = (int32_t*)malloc(sizeof(int32_t) * (size_t)n_ids);
  int32_t k = 0;
  for (char* p = b;; ++p) {
    if (*p == ' ' || *p == '\0') {
      const char end = *p;
      *p = '\0';
      const int32_t id = lookup(tok, n_tok, b);
      ids[k++] = id >= 0 ? id : unk;
      if (end == '\0') break;
      b = p + 1;
    }
  }
  void* al = fa_align_init(argv[1], 0, FA_GEMM_F16X3);
  if (!al) {
    fprintf(stderr, "init failed: %s\n", fa_offline_last_error());
    return 1;
  }
  const FaAudioFormat fmt = {f32 ? 0 : 1, 1, rate, FA_RESAMPLE_LOADER};
  const void* bufs[1] = {pcm};
  const int64_t frames = pcm_bytes / (f32 ? 4 : 2);
  const int32_t* id_rows[1] = {ids};
  void* r = fa_align_infer(al, bufs, &frames, 1, &fmt, id_rows, &n_ids);
  if (!r) {
    fprintf(stderr, "fa_align_infer failed: %s\n", fa_offline_last_error());
    return 1;
  }
  int32_t n_st = 0, n_kept = 0;
  const int32_t* st = fa_offline_result_stamps(r, 0, &n_st);
  const int32_t* kept = fa_offline_result_ids(r, 0, &n_kept);
  for (int32_t s = 0; s < n_st; ++s)   /* a stamp past the token list (a span after the last token) has no token */
    printf("%s %d %d\n", s < n_kept ? tok[kept[s]] : "-", st[2 * s], st[2 * s + 1]);
  fa_offline_free_result(r);
  fa_align_uninit(al);
  free(ids);
  free(pcm);
  free(text);
  free(tok);
  free(token_text);
  return 0;
}
