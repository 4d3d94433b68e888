/* Minimal C client of the handle-style API (include/funasr_b200.h): the call sequence a C/C++ server would use in place of
 * FunOfflineInit / FunOfflineInferBuffer / FunASRGetResult (runtime/onnxruntime/include/funasrruntime.h:100-116).
 *
 *   gcc -std=c99 -Iinclude examples/offline_demo.c -Lfunasr_b200 -lfunasr_b200 -Wl,-rpath,$PWD/funasr_b200 -o offline_demo
 *   ./offline_demo model.fab2 audio.pcm [rate]  (audio.pcm: mono s16le, 16 kHz unless rate says otherwise; model.fab2 from
 *                                               funasr_b200/pack.py)
 * At 16 kHz it calls fa_offline_infer; at any other rate fa_offline_infer_audio, which resamples on the GPU with the C++ runtime's
 * LinearResample (FA_RESAMPLE_RUNTIME).
 */
#include <stdio.h>
#include <stdlib.h>
#include "funasr_b200.h"

int main(int argc, char** argv) {
  printf("library: %s\n", fa_version());
  if (argc < 3) {
    void* h = fa_offline_init(argc > 1 ? argv[1] : "/nonexistent.fab2", 0, FA_GEMM_F16X3);
    if (!h) { printf("init failed (expected without a model / GPU): %s\n", fa_offline_last_error()); return 0; }
    fa_offline_uninit(h);
    return 0;
  }
  void* h = fa_offline_init(argv[1], 0, FA_GEMM_F16X3);
  if (!h) { fprintf(stderr, "init: %s\n", fa_offline_last_error()); return 1; }
  FILE* f = fopen(argv[2], "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", argv[2]); return 1; }
  fseek(f, 0, SEEK_END);
  long bytes = ftell(f);
  fseek(f, 0, SEEK_SET);
  short* pcm = (short*)malloc((size_t)bytes);
  if (fread(pcm, 1, (size_t)bytes, f) != (size_t)bytes) { fprintf(stderr, "short read\n"); return 1; }
  fclose(f);
  const void* bufs[1] = {pcm};
  int64_t n[1] = {bytes / 2};
  const int rate = argc > 3 ? atoi(argv[3]) : 16000;
  const FaAudioFormat fmt = {/*sample_format=*/1, /*channels=*/1, rate, FA_RESAMPLE_RUNTIME};
  void* r = rate == 16000 ? fa_offline_infer(h, bufs, n, 1, /*pcm_format=*/1) : fa_offline_infer_audio(h, bufs, n, 1, &fmt, NULL, 0, NULL, NULL);
  if (!r) { fprintf(stderr, "infer: %s\n", fa_offline_last_error()); return 1; }
  int32_t k = 0;
  const int32_t* ids = fa_offline_result_ids(r, 0, &k);
  printf("%.2f s of audio -> %d tokens:", fa_offline_result_audio_seconds(r), k);
  for (int i = 0; i < k; ++i) printf(" %d", ids[i]);
  printf("\n");
  fa_offline_free_result(r);
  fa_offline_uninit(h);
  free(pcm);
  return 0;
}
