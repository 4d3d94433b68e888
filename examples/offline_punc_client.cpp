// The call sequence of FunASR's own offline punctuation client (runtime/onnxruntime/bin/funasr-onnx-offline-punc.cpp) against this
// library: CTTransformerInit -> per line of a text file CTTransformerInfer -> CTTransformerGetResult -> CTTransformerFreeResult ->
// CTTransformerUninit; then, given an ASR model directory, one FunOfflineInit with "punc-dir" (and "vad-dir" when given) ->
// FunOfflineInfer -> FunASRGetResult / FunASRGetStamp / FunASRGetStampSents.
// Build (the header can be the reference's own funasrruntime.h: the signatures are identical):
//   g++ -std=c++17 -DFUNASR_RUNTIME_HEADER='"funasrruntime_b200.h"' -Iinclude examples/offline_punc_client.cpp -Lfunasr_b200 -lfunasr_b200
// usage: offline_punc_client <punc-model-dir> <text-file> [asr-model-dir audio.wav|audio.pcm [vad-model-dir [gemm-mode]]]
#ifndef FUNASR_RUNTIME_HEADER
#define FUNASR_RUNTIME_HEADER "funasrruntime_b200.h"
#endif
#include <stdint.h>
#include <stdio.h>
#include <fstream>
#include <string>      // before the runtime header: funasrruntime.h uses std::string without including <string> itself
#include FUNASR_RUNTIME_HEADER

int main(int argc, char** argv) {
  if (argc < 3) {
    fprintf(stderr, "usage: %s <punc-model-dir> <text-file> [asr-model-dir audio [vad-model-dir [gemm-mode]]]\n", argv[0]);
    return 2;
  }
  std::map<std::string, std::string> model_path;
  model_path.insert({"model-dir", argv[1]});
  FUNASR_HANDLE punc_handle = CTTransformerInit(model_path, 1);
  if (!punc_handle) { printf("punc init failed\n"); return 1; }
  std::ifstream in(argv[2]);
  std::string line;
  while (std::getline(in, line)) {
    FUNASR_RESULT result = CTTransformerInfer(punc_handle, line.c_str(), RASR_NONE, nullptr, PUNC_OFFLINE, nullptr);
    if (!result) { printf("no return data!\n"); return 1; }
    printf("punc_result %s\n", CTTransformerGetResult(result, 0));
    CTTransformerFreeResult(result);
  }
  CTTransformerUninit(punc_handle);
  if (argc < 5) return 0;
  std::map<std::string, std::string> asr_path;
  asr_path.insert({"model-dir", argv[3]});
  asr_path.insert({"punc-dir", argv[1]});
  if (argc > 5) asr_path.insert({"vad-dir", argv[5]});
  if (argc > 6) asr_path.insert({"gemm-mode", argv[6]});
  FUNASR_HANDLE asr_handle = FunOfflineInit(asr_path, 1, true, 1);
  if (!asr_handle) { printf("asr init failed\n"); return 1; }
  std::vector<std::vector<float>> hotwords_embedding;
  FUNASR_RESULT result = FunOfflineInfer(asr_handle, argv[4], RASR_NONE, nullptr, hotwords_embedding, 16000, true, nullptr);
  if (!result) { printf("no return data!\n"); return 1; }
  printf("asr_result %s\n", FunASRGetResult(result, 0));
  printf("asr_stamp %s\n", FunASRGetStamp(result));
  printf("asr_stamp_sents %s\n", FunASRGetStampSents(result));
  FunASRFreeResult(result);
  FunOfflineUninit(asr_handle);
  return 0;
}
