// The call sequence of FunASR's own throughput client (runtime/onnxruntime/bin/funasr-onnx-offline-rtf.cpp) against this library:
// one FunOfflineInit handle shared by N threads, each taking the next WAV of a list (FunASRWfstDecoderInit, CompileHotwordEmbedding,
// one warm-up FunOfflineInfer, then FunOfflineInfer -> FunASRGetResult / FunASRGetRetSnippetTime -> FunASRFreeResult per file), and
// the real-time factor of the whole run.  Concurrent calls on the one handle, with or without hotword rows, are pooled into shared GPU
// batches, each giving what it gives alone.
// Build (the header can be the reference's own funasrruntime.h: the signatures are identical):
//   g++ -std=c++17 -pthread -DFUNASR_RUNTIME_HEADER='"funasrruntime_b200.h"' -Iinclude examples/offline_rtf_client.cpp -Lfunasr_b200 -lfunasr_b200
// usage: offline_rtf_client <model-dir> <wav-list> <thread-num> [vad-model-dir|- [punc-model-dir|- [gemm-mode]]]
//   wav-list: one "<id> <path>" or "<path>" per line.  Prints "<id> <text>" per file in list order, then the RTF.
#ifndef FUNASR_RUNTIME_HEADER
#define FUNASR_RUNTIME_HEADER "funasrruntime_b200.h"
#endif
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <chrono>
#include <fstream>
#include <sstream>
#include <string>      // before the runtime header: funasrruntime.h uses std::string without including <string> itself
#include <thread>
#include <unordered_map>
#include <vector>
#include FUNASR_RUNTIME_HEADER

int main(int argc, char** argv) {
  if (argc < 4) {
    fprintf(stderr, "usage: %s <model-dir> <wav-list> <thread-num> [vad-model-dir|- [punc-model-dir|- [gemm-mode]]]\n", argv[0]);
    return 2;
  }
  std::map<std::string, std::string> model_path;
  model_path.insert({"model-dir", argv[1]});
  if (argc > 4 && std::string(argv[4]) != "-") model_path.insert({"vad-dir", argv[4]});
  if (argc > 5 && std::string(argv[5]) != "-") model_path.insert({"punc-dir", argv[5]});
  if (argc > 6) model_path.insert({"gemm-mode", argv[6]});
  const int thread_num = atoi(argv[3]) > 0 ? atoi(argv[3]) : 1;
  std::vector<std::string> ids, wavs;
  std::ifstream in(argv[2]);
  for (std::string line; std::getline(in, line);) {
    std::istringstream ss(line);
    std::string a, b;
    if (!(ss >> a)) continue;
    if (ss >> b) { ids.push_back(a); wavs.push_back(b); }
    else { ids.push_back(std::to_string(ids.size())); wavs.push_back(a); }
  }
  if (wavs.empty()) { printf("no wav\n"); return 1; }
  FUNASR_HANDLE asr_handle = FunOfflineInit(model_path, thread_num, true, 1);
  if (!asr_handle) { printf("asr init failed\n"); return 1; }
  std::vector<std::string> texts(wavs.size());
  std::vector<float> seconds(wavs.size(), 0.f);
  std::atomic<int> next(0), failed(0);
  auto run = [&]() {
    FUNASR_DEC_HANDLE decoder_handle = FunASRWfstDecoderInit(asr_handle, ASR_OFFLINE, 3.0f, 3.0f, 10.0f);
    std::unordered_map<std::string, int> hws_map;
    FunWfstDecoderLoadHwsRes(decoder_handle, 20, hws_map);
    std::string nn_hotwords;
    std::vector<std::vector<float>> hotwords_embedding = CompileHotwordEmbedding(asr_handle, nn_hotwords);
    FUNASR_RESULT warm = FunOfflineInfer(asr_handle, wavs[0].c_str(), RASR_NONE, nullptr, hotwords_embedding, 16000, true, decoder_handle);
    if (warm) FunASRFreeResult(warm);
    for (int i; (i = next.fetch_add(1)) < (int)wavs.size();) {
      FUNASR_RESULT result = FunOfflineInfer(asr_handle, wavs[i].c_str(), RASR_NONE, nullptr, hotwords_embedding, 16000, true, decoder_handle);
      if (!result) { ++failed; continue; }
      texts[i] = FunASRGetResult(result, 0);
      seconds[i] = FunASRGetRetSnippetTime(result);
      FunASRFreeResult(result);
    }
    FunWfstDecoderUnloadHwsRes(decoder_handle);
    FunASRWfstDecoderUninit(decoder_handle);
  };
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<std::thread> threads;
  for (int k = 0; k < thread_num; ++k) threads.emplace_back(run);
  for (auto& t : threads) t.join();
  const double wall = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  double audio = 0.0;
  for (size_t i = 0; i < wavs.size(); ++i) {
    printf("%s %s\n", ids[i].c_str(), texts[i].c_str());
    audio += seconds[i];
  }
  printf("threads %d files %zu failed %d audio %.3f s wall %.3f s rtf %.5f\n", thread_num, wavs.size(), failed.load(), audio, wall,
         audio > 0 ? wall / audio : 0.0);
  FunOfflineUninit(asr_handle);
  return failed.load() ? 1 : 0;
}
