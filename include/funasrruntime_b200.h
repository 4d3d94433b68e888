/* The OfflineStream surface of FunASR's C++ runtime — runtime/onnxruntime/include/funasrruntime.h:21-77,100-116 — with the SAME
 * names, argument lists and defaults, implemented over this library's handle API (funasr_b200.h: fa_offline_*).  A server written
 * against funasrruntime.h (runtime/websocket, runtime/http, bin/funasr-onnx-offline.cpp) links against libfunasr_b200.so with this
 * header in place of the original for the offline ASR calls it makes.  One handle may be shared by any number of threads, as the
 * reference's servers share it among their decoder threads: FunOfflineInfer / FunOfflineInferBuffer, CompileHotwordEmbedding,
 * FsmnVad* and CTTransformer* are safe on shared handles (funasr_b200.h, "Threads"); FunOfflineInfer* calls from many threads on
 * one handle are decoded together in shared GPU packs, with or without hotword rows, each giving what it gives alone, and their
 * punctuation ("punc-dir") and CTTransformerInfer calls on one handle share lockstep steps, each text punctuated as it is alone.
 * CompileHotwordEmbedding returns one zero row of 512 for a model without a hotword branch (Paraformer, BiCif), as the reference
 * does, so a server that decodes only when the embedding is non-empty decodes; the row is not used.  thread_num and batch_size stay ignored:
 * segments are packed by "batch-size-s".
 * Differences, all at run time, none in the signatures:
 *   model_path["model-dir"] names a directory holding `model.fab2` (funasr_b200/pack.py, written from an unmodified model.pt +
 *   am.mvn) and optionally `tokens.txt` (one token per line; without it results carry the token ids in decimal);
 *   optional keys "gemm-mode" (fp32 | fp16 | fp16x3 | fp16x6, default fp16x3) and "gpu-id" (default 0);
 *   there is no CPU path (use_gpu is ignored); the WFST / LM decoder entry points are accepted and ignored (greedy decoding, like
 *   the reference without --lm-dir).
 *   Audio at any sampling_rate from 1 000 to 192 000 Hz ("pcm" s16le mono; a WAV file or "wav" buffer at its header's rate, mono s16
 *   or float32) is resampled to 16 kHz on the GPU with the runtime's own LinearResample (FA_RESAMPLE_RUNTIME, as Audio::WavResample
 *   applies it), in FunOfflineInfer / FunOfflineInferBuffer with or without "vad-dir" and in FsmnVadInfer / FsmnVadInferBuffer.  One
 *   known difference: the runtime decodes "wav" buffers with ffmpeg (swresample) where it is built with it; here they take
 *   LinearResample too.
 *   model_path["vad-dir"] (optional) names a directory holding `vad.fab2` (funasr_b200/pack.py: write_vad_model_file, from the FSMN-VAD
 *   model.pt + am.mvn + the model_conf of its config.yaml).  With it FunOfflineInfer / FunOfflineInferBuffer segment the audio first
 *   (fa_offline_infer_vad) with the runtime's semantics: a FIXED end silence (the file's max_end_silence_time, fsmn-vad.cpp), segment
 *   texts concatenated in time order (funasrruntime.cpp:287-296); optional key "batch-size-s" sets the segment packing (default 300).
 *   Without it a buffer is decoded as one utterance, as before.
 *   model_path["punc-dir"] (optional) names a directory holding `punc.fab2` (funasr_b200/pack.py: write_punc_model_file, from the
 *   CT-Transformer model.pt + its punc_list / token_list + config).  With it FunOfflineInfer / FunOfflineInferBuffer punctuate each
 *   result text after the join, with or without "vad-dir" (funasrruntime.cpp:311-314); without it results are unpunctuated, as before.
 *   The punctuation is the Python model's (CTTransformer.inference): its word split, exact lookup with <unk>, 20-word windows with the
 *   unfinished tail carried over and a long window cut at its last comma when the comma lies at index 2 or later.  The runtime's own
 *   AddPunc (ct-transformer.cpp) differs: it has its own tokenizer and cuts at any comma with nLastCommaIndex > 0.  This library keeps
 *   one definition, as it does for stamps.  ITN is not provided (itn is ignored).
 *   With "punc-dir" and a BiCif model FunASRGetStampSents is the runtime's TimestampSentence (util.cpp:569-637) over the punctuated
 *   text and the FunASRGetStamp pairs; without "punc-dir" it stays empty.
 *   A SenseVoiceSmall `model.fab2` (funasr_b200/pack.py: write_sensevoice_model_file) makes a SenseVoice handle: the file decides
 *   the model kind (the runtime decides by "SenseVoiceSmall" in the directory name).  FunOfflineInferBuffer maps svs_lang through the
 *   runtime's lid_map (an unknown name is "auto") and svs_itn to text norm 14 / 15; FunOfflineInfer uses "auto" / true.  The text is
 *   the runtime's CTCSearch over the ids and tokens.txt, except that with exactly 3 ids the fourth tag is empty (the runtime reads one
 *   past its vector there); the ids are the Python model's arg-max of log_softmax.  With "vad-dir" segment texts are concatenated
 *   without a separator; "punc-dir" and ITN are ignored, FunASRGetStamp / FunASRGetStampSents stay empty, and CompileHotwordEmbedding
 *   returns one zero row of 512.
 *   CTTransformerInit: model_path["model-dir"] holds `punc.fab2` ("gpu-id" as above); only PUNC_OFFLINE is provided (PUNC_ONLINE is
 *   refused with a FunB200LastError message); CTTransformerGetResult ignores n_index, as the runtime does.
 *   FsmnVadInit: model_path["model-dir"] holds `vad.fab2` ("gpu-id" as above); FsmnVadInferBuffer is offline only (input_finished
 *   must be true) and takes "pcm" (s16le) or "wav" (PCM16 / float32); FsmnVadOnlineInit is not provided.
 */
#pragma once
#include <stdint.h>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#define _FUNASRAPI

typedef void* FUNASR_HANDLE;
typedef void* FUNASR_RESULT;
typedef void* FUNASR_DEC_HANDLE;
typedef unsigned char FUNASR_BOOL;

#define FUNASR_TRUE 1
#define FUNASR_FALSE 0
#define QM_DEFAULT_THREAD_NUM 4

typedef enum { RASR_NONE = -1, RASRM_CTC_GREEDY_SEARCH = 0, RASRM_CTC_RPEFIX_BEAM_SEARCH = 1, RASRM_ATTENSION_RESCORING = 2 } FUNASR_MODE;
typedef enum { ASR_OFFLINE = 0, ASR_ONLINE = 1, ASR_TWO_PASS = 2 } ASR_TYPE;
typedef enum { PUNC_OFFLINE = 0, PUNC_ONLINE = 1 } PUNC_TYPE;

typedef void (*QM_CALLBACK)(int cur_step, int n_total);

// OfflineStream (funasrruntime.h:100-116)
_FUNASRAPI FUNASR_HANDLE FunOfflineInit(std::map<std::string, std::string>& model_path, int thread_num, bool use_gpu = false, int batch_size = 1);
_FUNASRAPI void FunOfflineReset(FUNASR_HANDLE handle, FUNASR_DEC_HANDLE dec_handle = nullptr);
_FUNASRAPI FUNASR_RESULT FunOfflineInferBuffer(FUNASR_HANDLE handle, const char* sz_buf, int n_len, FUNASR_MODE mode, QM_CALLBACK fn_callback,
                                               const std::vector<std::vector<float>>& hw_emb, int sampling_rate = 16000,
                                               std::string wav_format = "pcm", bool itn = true, FUNASR_DEC_HANDLE dec_handle = nullptr,
                                               std::string svs_lang = "auto", bool svs_itn = true);
_FUNASRAPI FUNASR_RESULT FunOfflineInfer(FUNASR_HANDLE handle, const char* sz_filename, FUNASR_MODE mode, QM_CALLBACK fn_callback,
                                         const std::vector<std::vector<float>>& hw_emb, int sampling_rate = 16000, bool itn = true,
                                         FUNASR_DEC_HANDLE dec_handle = nullptr);
_FUNASRAPI const std::vector<std::vector<float>> CompileHotwordEmbedding(FUNASR_HANDLE handle, std::string& hotwords, ASR_TYPE mode = ASR_OFFLINE);
_FUNASRAPI void FunOfflineUninit(FUNASR_HANDLE handle);

// result accessors shared with the other streams (funasrruntime.h:67-77)
_FUNASRAPI const char* FunASRGetResult(FUNASR_RESULT result, int n_index);
_FUNASRAPI const char* FunASRGetStamp(FUNASR_RESULT result);
_FUNASRAPI const char* FunASRGetStampSents(FUNASR_RESULT result);
_FUNASRAPI const int FunASRGetRetNumber(FUNASR_RESULT result);
_FUNASRAPI void FunASRFreeResult(FUNASR_RESULT result);
_FUNASRAPI const float FunASRGetRetSnippetTime(FUNASR_RESULT result);

// VAD (funasrruntime.h:81-91, without FsmnVadOnlineInit)
_FUNASRAPI FUNASR_HANDLE FsmnVadInit(std::map<std::string, std::string>& model_path, int thread_num);
_FUNASRAPI FUNASR_RESULT FsmnVadInferBuffer(FUNASR_HANDLE handle, const char* sz_buf, int n_len, QM_CALLBACK fn_callback, bool input_finished = true,
                                            int sampling_rate = 16000, std::string wav_format = "pcm");
_FUNASRAPI FUNASR_RESULT FsmnVadInfer(FUNASR_HANDLE handle, const char* sz_filename, QM_CALLBACK fn_callback, int sampling_rate = 16000);
_FUNASRAPI std::vector<std::vector<int>>* FsmnVadGetResult(FUNASR_RESULT result, int n_index);
_FUNASRAPI void FsmnVadFreeResult(FUNASR_RESULT result);
_FUNASRAPI void FsmnVadUninit(FUNASR_HANDLE handle);
_FUNASRAPI const float FsmnVadGetRetSnippetTime(FUNASR_RESULT result);

// punctuation (funasrruntime.h:94-98), offline only
_FUNASRAPI FUNASR_HANDLE CTTransformerInit(std::map<std::string, std::string>& model_path, int thread_num, PUNC_TYPE type = PUNC_OFFLINE);
_FUNASRAPI FUNASR_RESULT CTTransformerInfer(FUNASR_HANDLE handle, const char* sz_sentence, FUNASR_MODE mode, QM_CALLBACK fn_callback,
                                            PUNC_TYPE type = PUNC_OFFLINE, FUNASR_RESULT pre_result = nullptr);
_FUNASRAPI const char* CTTransformerGetResult(FUNASR_RESULT result, int n_index);
_FUNASRAPI void CTTransformerFreeResult(FUNASR_RESULT result);
_FUNASRAPI void CTTransformerUninit(FUNASR_HANDLE handle);

// WFST decoder (funasrruntime.h:134-138): accepted, no effect (greedy decoding)
_FUNASRAPI FUNASR_DEC_HANDLE FunASRWfstDecoderInit(FUNASR_HANDLE handle, int asr_type, float glob_beam, float lat_beam, float am_scale);
_FUNASRAPI void FunASRWfstDecoderUninit(FUNASR_DEC_HANDLE handle);
_FUNASRAPI void FunWfstDecoderLoadHwsRes(FUNASR_DEC_HANDLE handle, int inc_bias, std::unordered_map<std::string, int>& hws_map);
_FUNASRAPI void FunWfstDecoderUnloadHwsRes(FUNASR_DEC_HANDLE handle);

// extension (not in funasrruntime.h): why the last call on this thread failed
const char* FunB200LastError();
