// The call sequence of FunASR's own offline VAD client (runtime/onnxruntime/bin/funasr-onnx-offline-vad.cpp:61-157) against this
// library: FsmnVadInit -> FsmnVadInfer (file) / FsmnVadInferBuffer -> FsmnVadGetResult / FsmnVadGetRetSnippetTime -> FsmnVadFreeResult
// -> FsmnVadUninit; then, given an ASR model directory, one FunOfflineInit with "vad-dir" -> FunOfflineInfer -> FunASRGetResult, the
// whole recording segmented by the VAD and decoded segment by segment.
// Build (the header can be the reference's own funasrruntime.h: the signatures are identical):
//   g++ -std=c++17 -DFUNASR_RUNTIME_HEADER='"funasrruntime_b200.h"' -Iinclude examples/offline_vad_client.cpp -Lfunasr_b200 -lfunasr_b200
// usage: offline_vad_client <vad-model-dir> <audio.wav|audio.pcm> [asr-model-dir [gemm-mode [batch-size-s]]]
#ifndef FUNASR_RUNTIME_HEADER
#define FUNASR_RUNTIME_HEADER "funasrruntime_b200.h"
#endif
#include <stdint.h>
#include <stdio.h>
#include <fstream>
#include <sstream>
#include <string>      // before the runtime header: funasrruntime.h uses std::string without including <string> itself
#include FUNASR_RUNTIME_HEADER

static void print_segs(const char* what, std::vector<std::vector<int>>* segs) {
  printf("%s", what);
  for (const auto& s : *segs) printf(" [%d,%d]", s[0], s[1]);
  printf("\n");
}

int main(int argc, char** argv) {
  if (argc < 3) {
    fprintf(stderr, "usage: %s <vad-model-dir> <audio.wav|audio.pcm> [asr-model-dir [gemm-mode [batch-size-s]]]\n", argv[0]);
    return 2;
  }
  std::map<std::string, std::string> model_path;
  model_path.insert({"model-dir", argv[1]});
  model_path.insert({"quantize", "false"});
  FUNASR_HANDLE vad_handle = FsmnVadInit(model_path, 1);
  if (!vad_handle) { fprintf(stderr, "FsmnVad init failed\n"); return 1; }
  float snippet_time = 0.f;
  // 1) the file entry point
  FUNASR_RESULT result = FsmnVadInfer(vad_handle, argv[2], nullptr, 16000);
  if (!result) { fprintf(stderr, "no return data!\n"); return 1; }
  print_segs("file_segments", FsmnVadGetResult(result, 0));
  snippet_time += FsmnVadGetRetSnippetTime(result);
  FsmnVadFreeResult(result);
  // 2) the buffer entry point with the same bytes
  std::ifstream f(argv[2], std::ios::binary);
  std::stringstream ss;
  ss << f.rdbuf();
  const std::string bytes = ss.str();
  const std::string name = argv[2];
  const bool wav = name.size() > 4 && name.compare(name.size() - 4, 4, ".wav") == 0;
  result = FsmnVadInferBuffer(vad_handle, bytes.data(), (int)bytes.size(), nullptr, true, 16000, wav ? "wav" : "pcm");
  if (!result) { fprintf(stderr, "no return data!\n"); return 1; }
  print_segs("buffer_segments", FsmnVadGetResult(result, 0));
  snippet_time += FsmnVadGetRetSnippetTime(result);
  FsmnVadFreeResult(result);
  printf("audio_seconds %.3f\n", snippet_time);
  FsmnVadUninit(vad_handle);
  if (argc < 4) return 0;
  // 3) recognition of the whole recording, segmented by the same VAD model
  std::map<std::string, std::string> asr_path;
  asr_path.insert({"model-dir", argv[3]});
  asr_path.insert({"vad-dir", argv[1]});
  if (argc > 4) asr_path.insert({"gemm-mode", argv[4]});
  if (argc > 5) asr_path.insert({"batch-size-s", argv[5]});
  FUNASR_HANDLE asr_handle = FunOfflineInit(asr_path, 1, true, 1);
  if (!asr_handle) { fprintf(stderr, "FunASR init failed\n"); return 1; }
  std::vector<std::vector<float>> hotwords_embedding;
  result = FunOfflineInfer(asr_handle, argv[2], RASR_NONE, nullptr, hotwords_embedding, 16000, true, nullptr);
  if (!result) { fprintf(stderr, "no return data!\n"); return 1; }
  printf("asr_result %s\n", FunASRGetResult(result, 0));
  printf("asr_seconds %.3f\n", FunASRGetRetSnippetTime(result));
  FunASRFreeResult(result);
  FunOfflineUninit(asr_handle);
  return 0;
}
