// The call sequence of FunASR's own offline client (runtime/onnxruntime/bin/funasr-onnx-offline.cpp) on a SenseVoiceSmall model
// directory, with the query the websocket servers pass from each client message (runtime/websocket/bin/websocket-server.cpp:365-391):
// FunOfflineInit -> CompileHotwordEmbedding -> FunOfflineInferBuffer(..., svs_lang, svs_itn) -> FunASRGetResult / FunASRGetStamp /
// FunASRGetStampSents -> FunASRFreeResult -> FunOfflineUninit.
// Build (the header can be the reference's own funasrruntime.h: the signatures are identical):
//   g++ -std=c++17 -DFUNASR_RUNTIME_HEADER='"funasrruntime_b200.h"' -Iinclude examples/offline_sv_client.cpp -Lfunasr_b200 -lfunasr_b200
// usage: offline_sv_client <model-dir> <audio.wav|audio.pcm> [svs_lang [svs_itn 0|1 [vad-dir|- [punc-dir|- [gemm-mode]]]]]
#ifndef FUNASR_RUNTIME_HEADER
#define FUNASR_RUNTIME_HEADER "funasrruntime_b200.h"
#endif
#include <stdint.h>
#include <stdio.h>
#include <fstream>
#include <sstream>
#include <string>      // before the runtime header: funasrruntime.h uses std::string without including <string> itself
#include FUNASR_RUNTIME_HEADER

int main(int argc, char** argv) {
  if (argc < 3) {
    fprintf(stderr, "usage: %s <model-dir> <audio.wav|audio.pcm> [svs_lang [svs_itn 0|1 [vad-dir|- [punc-dir|- [gemm-mode]]]]]\n", argv[0]);
    return 2;
  }
  const std::string svs_lang = argc > 3 ? argv[3] : "auto";
  const bool svs_itn = argc > 4 ? std::string(argv[4]) != "0" : true;
  std::map<std::string, std::string> model_path;
  model_path.insert({"model-dir", argv[1]});
  if (argc > 5 && std::string(argv[5]) != "-") model_path.insert({"vad-dir", argv[5]});
  if (argc > 6 && std::string(argv[6]) != "-") model_path.insert({"punc-dir", argv[6]});
  if (argc > 7) model_path.insert({"gemm-mode", argv[7]});
  FUNASR_HANDLE asr_handle = FunOfflineInit(model_path, 1, true, 1);
  if (!asr_handle) { printf("asr init failed\n"); return 1; }
  std::string hotwords;
  std::vector<std::vector<float>> hotwords_embedding = CompileHotwordEmbedding(asr_handle, hotwords);
  std::ifstream f(argv[2], std::ios::binary);
  if (!f) { printf("cannot open %s\n", argv[2]); return 1; }
  std::stringstream ss;
  ss << f.rdbuf();
  const std::string bytes = ss.str();
  const std::string name = argv[2];
  const bool wav = name.size() > 4 && name.compare(name.size() - 4, 4, ".wav") == 0;
  FUNASR_RESULT result = FunOfflineInferBuffer(asr_handle, bytes.data(), (int)bytes.size(), RASR_NONE, nullptr, hotwords_embedding, 16000,
                                               wav ? "wav" : "pcm", true, nullptr, svs_lang, svs_itn);
  if (!result) { printf("no return data!\n"); return 1; }
  printf("hotword_rows %d\n", (int)hotwords_embedding.size());
  printf("asr_result %s\n", FunASRGetResult(result, 0));
  printf("asr_stamp %s\n", FunASRGetStamp(result));
  printf("asr_stamp_sents %s\n", FunASRGetStampSents(result));
  FunASRFreeResult(result);
  FunOfflineUninit(asr_handle);
  return 0;
}
