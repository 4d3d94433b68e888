/* Long-audio recognition with speaker labels through the plain C handle API: FSMN-VAD segments, Paraformer ids per recording and one
 * CAM++ speaker per segment (LongAudioPipeline.generate with spk_model, vad_segment mode).
 * Model files: funasr_b200/pack.py write_model_file, write_vad_model_file and write_campplus_model_file.
 * Build:  cc -std=c99 -Iinclude examples/offline_spk_client.c -Lfunasr_b200 -lfunasr_b200 -o offline_spk_client
 * usage:  offline_spk_client <asr.fab2> <vad.fab2> <spk.fab2> <audio.pcm (s16le, 16 kHz)> [preset_spk_num] */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "funasr_b200.h"

static int16_t* read_pcm(const char* path, int64_t* n) {
  FILE* f = fopen(path, "rb");
  if (!f) return NULL;
  fseek(f, 0, SEEK_END);
  const long bytes = ftell(f);
  rewind(f);
  int16_t* pcm = (int16_t*)malloc(bytes > 0 ? (size_t)bytes : 1);
  *n = pcm ? (int64_t)fread(pcm, 2, (size_t)bytes / 2, f) : 0;
  fclose(f);
  return pcm;
}

int main(int argc, char** argv) {
  if (argc < 5) {
    fprintf(stderr, "usage: %s <asr.fab2> <vad.fab2> <spk.fab2> <audio.pcm> [preset_spk_num]\n", argv[0]);
    return 2;
  }
  const int32_t preset = argc > 5 ? atoi(argv[5]) : 0;
  void* asr = fa_offline_init(argv[1], 0, FA_GEMM_F16X3);
  void* vad = asr ? fa_vad_init(argv[2], 0) : NULL;
  void* spk = vad ? fa_spk_init(argv[3], 0, FA_GEMM_F16X3) : NULL;
  if (!spk) {
    fprintf(stderr, "init failed: %s\n", fa_offline_last_error());
    return 1;
  }
  int64_t n = 0;
  int16_t* pcm = read_pcm(argv[4], &n);
  if (!pcm) {
    fprintf(stderr, "cannot read %s\n", argv[4]);
    return 1;
  }
  const void* bufs[1] = {pcm};
  void* r = fa_offline_infer_vad_spk(asr, vad, spk, bufs, &n, 1, /*pcm_format s16le*/ 1, NULL, 0, NULL, NULL, NULL, preset);
  if (!r) {
    fprintf(stderr, "fa_offline_infer_vad_spk failed: %s\n", fa_offline_last_error());
    return 1;
  }
  int32_t n_seg = 0, n_spk = 0;
  const int32_t* seg = fa_offline_result_segments(r, 0, &n_seg);
  const int32_t* who = fa_offline_result_spk(r, 0, &n_spk);
  for (int32_t s = 0; s < n_seg; ++s)
    printf("[%d, %d] ms  %d tokens  speaker %d\n", seg[3 * s], seg[3 * s + 1], seg[3 * s + 2], s < n_spk ? who[s] : -1);
  fa_offline_free_result(r);
  free(pcm);
  fa_spk_uninit(spk);
  fa_vad_uninit(vad);
  fa_offline_uninit(asr);
  return 0;
}
