"""GPU: SenseVoiceSmall through the C handle API (fa_offline_infer_sv, fa_offline_infer_vad_sv, fa_sv_query_rows) and the C++ runtime
surface (FunOfflineInferBuffer with svs_lang / svs_itn), against the reference's goldens and bit for bit against SenseVoiceEngine /
LongAudioPipeline with SenseVoiceSmallB200 run in the same mode."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, load_sv_case

import funasr_b200
from funasr_b200 import _abi, pack, synth
from funasr_b200.engine import SenseVoiceEngine
from funasr_b200.modules import SenseVoiceSmallB200
from funasr_b200.offline import OfflineRecognizer, OfflineVad
from test_offline_punc_host import ENC_CONF as PUNC_ENC_CONF
from test_offline_sv_host import ctc_search_text
from test_offline_vad_gpu import _CountingAsr, _python_result, _s16, _vad_plugin, _wav_bytes

DEV = "cuda:0"
LID, TN = SenseVoiceSmallB200.lid_dict, SenseVoiceSmallB200.textnorm_dict
# golden -> (SV_CASES entry whose waveforms and weights it uses, language, use_itn); the query goldens: oracle/make_sv_query_golden.py
GOLD_CASES = {"sv_tiny_ragged3": ("sv_tiny_ragged3", "auto", False), "sv_large_single": ("sv_large_single", "auto", False),
              "sv_tiny_en_itn": ("sv_tiny_ragged3", "en", True), "sv_tiny_yue_woitn": ("sv_tiny_ragged3", "yue", False)}
# must match oracle/make_sv_query_golden.py:LONG_SV_CASES / LONG_SV_WEIGHT_SEED
LONG_SV = (40.0, 7, [(3.0, 2.5), (1.5, 2.2), (4.0, 3.0), (2.0, 2.2), (6.0, 2.4)])
LONG_SV_WEIGHT_SEED = 6
LONG_KW = {"batch_size_s": 6, "language": "zh", "use_itn": True}


def _gold(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


_FILES = {}


def _sv_file(tmp_path_factory, case):
    """(model file, cfg, state, cmvn, wavs) of an SV_CASES entry; one file per case for the module."""
    if case not in _FILES:
        cfg, wseed, wavs, cmvn, _ = load_sv_case(case)
        state = synth.make_sensevoice_state_dict(cfg, wseed)
        path = str(tmp_path_factory.mktemp("sv") / "model.fab2")
        pack.write_sensevoice_model_file(path, state, cfg, cmvn)
        _FILES.clear()                                                   # at most one (large ~1 GB) state alive
        _FILES[case] = (path, cfg, state, cmvn, wavs)
    return _FILES[case]


@pytest.fixture(scope="module")
def tiny(tmp_path_factory):
    return _sv_file(tmp_path_factory, "sv_tiny_ragged3")


@pytest.fixture(scope="module")
def vad_file(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("vad") / "vad.fab2")
    pack.write_vad_model_file(path, synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    return path


def _engine_ids(eng, wavs, lang, tn):
    lens = [int(w.numel()) for w in wavs]
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
    return eng.forward_wav(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), lens, language_id=lang, textnorm_id=tn)["ids"]


def _np(wavs):
    return [w.numpy().astype(np.float32) for w in wavs]


# ------------------------------------------------------------------------------------------------------------ goldens
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3", "fp16x6"])
@pytest.mark.parametrize("name", list(GOLD_CASES))
def test_handle_vs_reference_goldens(tmp_path_factory, name, mode):
    """Float32 input: the handle's ids equal the unmodified reference's SenseVoiceSmall.inference bit for bit for every query the goldens
    cover.  s16 input: equal to SenseVoiceEngine fed the same quantised waveforms."""
    case, language, use_itn = GOLD_CASES[name]
    path, cfg, state, cmvn, wavs = _sv_file(tmp_path_factory, case)
    g = _gold(name)
    rec = OfflineRecognizer(path, 0, mode)
    assert rec.is_sensevoice and not rec.has_timestamps
    got = rec.infer(_np(wavs), language=language, use_itn=use_itn)
    assert [t for r in got for t in r] == g["ids_flat"].tolist()
    assert [len(r) for r in got] == g["ids_len"].tolist()
    assert [(1 + (w.numel() - 400) // 160 + 5) // 6 + 4 for w in wavs] == g["enc_lens"].tolist()     # LFR frames + the 4 query rows
    pcm = [_s16(w) for w in _np(wavs)]
    eng = SenseVoiceEngine(state, cfg, DEV, gemm_mode=mode, cmvn=cmvn)
    want = _engine_ids(eng, [torch.from_numpy(p.astype(np.float32) / 32768.0) for p in pcm], LID[language], TN["withitn" if use_itn else "woitn"])
    assert rec.infer(pcm, language=language, use_itn=use_itn) == want
    rec.close()


@pytest.mark.gpu
def test_every_query_equals_the_engine(tiny):
    path, cfg, state, cmvn, wavs = tiny
    rec = OfflineRecognizer(path, 0, "fp16x3")
    eng = SenseVoiceEngine(state, cfg, DEV, gemm_mode="fp16x3", cmvn=cmvn)
    outs = set()
    for language, lid in LID.items():
        for use_itn in (True, False):
            got = rec.infer(_np(wavs), language=language, use_itn=use_itn)
            assert got == _engine_ids(eng, wavs, lid, TN["withitn" if use_itn else "woitn"]), (language, use_itn)
            outs.add(str(got))
    assert len(outs) > 1                                                 # the query reaches the result
    rec.close()


@pytest.mark.gpu
def test_mixed_languages_in_one_batch(tiny):
    path, cfg, state, cmvn, wavs = tiny
    rec = OfflineRecognizer(path, 0, "fp16x3")
    x = _np(wavs)
    for langs, itns in ((["zh", "en", "yue"], [True, False, True]), (["ja", "auto", "ko"], [False, True, False])):
        mixed = rec.infer(x, language=langs, use_itn=itns)
        for b in range(len(x)):
            assert mixed[b] == rec.infer(x, language=langs[b], use_itn=itns[b])[b]
    rec.close()


@pytest.mark.gpu
def test_query_rows_kernel_bit_exact():
    """fa_sv_query_rows against index_select into a strided buffer; every other row keeps its sentinel."""
    lib = _abi.load()
    g = torch.Generator().manual_seed(3)
    n_embed, cols, B, stride = 16, 560, 5, 9
    embed = torch.randn(n_embed, cols, generator=g).to(DEV)
    ids = torch.tensor([[0, 15], [3, 14], [13, 15], [7, 14], [12, 15]], dtype=torch.int32, device=DEV)
    dst = torch.full((B, stride, cols), 7.25, device=DEV)
    _abi.check(lib.fa_sv_query_rows(embed.data_ptr(), n_embed, cols, ids.data_ptr(), B, dst.data_ptr(), stride,
                                    torch.cuda.current_stream().cuda_stream), "fa_sv_query_rows")
    torch.cuda.synchronize()
    for b in range(B):
        q = torch.tensor([int(ids[b, 0]), 1, 2, int(ids[b, 1])], device=DEV)
        assert torch.equal(dst[b, :4], embed.index_select(0, q))
        assert bool((dst[b, 4:] == 7.25).all())
    assert lib.fa_sv_query_rows(embed.data_ptr(), n_embed, cols, ids.data_ptr(), B, dst.data_ptr(), 3, None) != _abi.FA_OK


# ------------------------------------------------------------------------------------------------------------ long audio
def _sv_pipeline(state, cfg, cmvn, mode):
    asr = SenseVoiceSmallB200(encoder="SenseVoiceEncoderSmallB200",
                              encoder_conf=dict(output_size=512, attention_heads=4, linear_units=2048, num_blocks=cfg.enc_layers,
                                                tp_blocks=cfg.tp_layers, input_layer="pe", kernel_size=11, sanm_shfit=0,
                                                selfattention_layer_type="sanm"), input_size=560, vocab_size=cfg.vocab, gemm_mode=mode)
    asr.load_state_dict(state, strict=True)
    asr.to(DEV).eval()
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0, cmvn=cmvn)
    vad, vad_fe = _vad_plugin()
    counting = _CountingAsr(asr)
    return funasr_b200.LongAudioPipeline(counting, fe, vad, vad_fe, device=DEV), counting


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_long_audio_vs_reference_golden_and_pipeline(tmp_path, vad_file, mode):
    cfg, _, _, cmvn, _ = load_sv_case("sv_tiny_ragged3")
    state = synth.make_sensevoice_state_dict(cfg, LONG_SV_WEIGHT_SEED)
    path = str(tmp_path / "model.fab2")
    pack.write_sensevoice_model_file(path, state, cfg, cmvn)
    g = _gold("longaudio_sv_40s")
    wav = synth.make_vad_wav(*LONG_SV).numpy()
    assert wav.size == int(g["n_samples"])
    rec, vad = OfflineRecognizer(path, 0, mode), OfflineVad(vad_file, 0)
    got = rec.infer_long([wav], vad, **LONG_KW)[0]
    assert got["vad_segments"] == g["segments"].tolist() and len(got["vad_segments"]) >= 2
    assert got["token_int"] == g["ids"].tolist()
    assert sum(got["n_tokens"]) == len(got["token_int"]) and "timestamp" not in got
    pipe, counting = _sv_pipeline(state, cfg, cmvn, mode)
    assert got == _python_result(pipe, counting, wav, **LONG_KW)
    kw = dict(LONG_KW, language="en", use_itn=False)
    assert rec.infer_long([wav], vad, **kw)[0] == _python_result(pipe, counting, wav, **kw)
    rec.close()
    vad.close()


@pytest.mark.gpu
def test_long_audio_three_recordings_equal_three_calls(tiny, vad_file):
    path = tiny[0]
    rec, vad = OfflineRecognizer(path, 0, "fp16x3"), OfflineVad(vad_file, 0)
    wavs = [synth.make_vad_wav(*LONG_SV).numpy(), synth.make_vad_wav(25.0, 8, [(2.0, 2.5), (3.0, 2.1)]).numpy(), synth.make_vad_wav(18.0, 21).numpy()]
    langs, itns = ["zh", "en", "auto"], [True, False, True]
    many = rec.infer_long(wavs, vad, batch_size_s=6, language=langs, use_itn=itns)
    assert many == [rec.infer_long([w], vad, batch_size_s=6, language=l, use_itn=i)[0] for w, l, i in zip(wavs, langs, itns)]
    # fa_offline_infer_vad on a SenseVoice handle: the defaults
    lib = rec.lib
    arr = [np.ascontiguousarray(w) for w in wavs[:1]]
    ptrs, lens = (C.c_void_p * 1)(arr[0].ctypes.data), (C.c_int64 * 1)(arr[0].size)
    r = lib.fa_offline_infer_vad(rec.handle, vad.handle, ptrs, lens, 1, 0, None, 0, None)
    assert r
    n = C.c_int32(0)
    p = lib.fa_offline_result_ids(r, 0, C.byref(n))
    assert [p[k] for k in range(n.value)] == rec.infer_long(wavs[:1], vad)[0]["token_int"]
    lib.fa_offline_free_result(r)
    with pytest.raises(_abi.FunasrB200Error, match="recording 1: language id 16"):
        bad = (C.c_int32 * 3)(0, 16, 0)
        ptrs3 = (C.c_void_p * 3)(*[np.ascontiguousarray(w).ctypes.data for w in wavs])
        lens3 = (C.c_int64 * 3)(*[w.size for w in wavs])
        opts = _abi.FaLongAudioOptions(300, 60, 0, 15, _abi.FaVadRunOptions(1, 0, float("nan")))
        if not lib.fa_offline_infer_vad_sv(rec.handle, vad.handle, ptrs3, lens3, 3, 0, bad, None, C.byref(opts)):
            raise _abi.FunasrB200Error(lib.fa_offline_last_error().decode())
    rec.close()
    vad.close()


# ------------------------------------------------------------------------------------------------------------ refusals
@pytest.mark.gpu
def test_refusals_and_defaults(tiny, tmp_path):
    path, cfg, state, cmvn, wavs = tiny
    rec = OfflineRecognizer(path, 0, "fp16x3")
    lib = rec.lib
    x = _np(wavs)
    ptrs = (C.c_void_p * 3)(*[a.ctypes.data for a in x])
    lens = (C.c_int64 * 3)(*[a.size for a in x])
    for lang, tn, msg in (([0, 0, 16], None, "utterance 2: language id 16"), ([0, -1, 0], None, "utterance 1: language id -1"),
                          (None, [15, 15, 99], "utterance 2: textnorm id 99")):
        la = None if lang is None else (C.c_int32 * 3)(*lang)
        ta = None if tn is None else (C.c_int32 * 3)(*tn)
        assert not lib.fa_offline_infer_sv(rec.handle, ptrs, lens, 3, 0, la, ta)
        assert msg in lib.fa_offline_last_error().decode()
    with pytest.raises(_abi.FunasrB200Error, match="400 samples"):
        rec.infer([x[0], x[1][:399]], language="zh")
    # NULL arrays, fa_offline_infer and fa_offline_infer_hw (hotwords ignored) all give the defaults "auto" / "woitn"
    want = rec.infer(x, language="auto", use_itn=False)
    r = lib.fa_offline_infer_sv(rec.handle, ptrs, lens, 3, 0, None, None)
    hw = np.ones((2, 512), np.float32)
    r2 = lib.fa_offline_infer_hw(rec.handle, ptrs, lens, 3, 0, hw.ctypes.data, 2)
    n = C.c_int32(0)
    for res in (r, r2):
        ids = []
        for i in range(3):
            p = lib.fa_offline_result_ids(res, i, C.byref(n))
            ids.append([p[k] for k in range(n.value)])
            assert not lib.fa_offline_result_stamps(res, i, C.byref(n)) and n.value == 0
        assert ids == want
        lib.fa_offline_free_result(res)
    assert rec.infer(x) == want
    # a Paraformer handle refuses the SenseVoice entry and the query keywords
    pcfg = synth.PARAFORMER_TINY
    ppath = str(tmp_path / "para.fab2")
    pack.write_model_file(ppath, synth.make_state_dict(pcfg, 3), pcfg, synth.make_cmvn(pcfg, 1))
    para = OfflineRecognizer(ppath, 0, "fp16x3")
    assert not para.is_sensevoice
    assert not lib.fa_offline_infer_sv(para.handle, ptrs, lens, 3, 0, None, None)
    assert "not a SenseVoice model file" in lib.fa_offline_last_error().decode()
    with pytest.raises(_abi.FunasrB200Error):
        para.infer(x, language="zh")
    para.close()
    rec.close()


# ------------------------------------------------------------------------------------------------------------ runtime shim
@pytest.mark.gpu
def test_runtime_client_svs_lang_and_itn(tiny, vad_file, tmp_path):
    """examples/offline_sv_client.cpp on a SenseVoice model-dir: FunASRGetResult is the runtime's CTCSearch text over the engine's ids
    (per segment, joined without a separator, with "vad-dir"), for svs_lang auto / zh / en and svs_itn true / false, with a "punc-dir"
    present (ignored for SenseVoice); FunASRGetStamp and FunASRGetStampSents stay empty."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    path, cfg, state, cmvn, wavs = tiny
    inc, libdir = os.path.join(ROOT, "include"), os.path.join(ROOT, "funasr_b200")
    exe = str(tmp_path / "sv_client")
    r = subprocess.run(["g++", "-std=c++17", '-DFUNASR_RUNTIME_HEADER="funasrruntime_b200.h"', "-I" + inc,
                        os.path.join(ROOT, "examples", "offline_sv_client.cpp"), "-L" + libdir, "-lfunasr_b200", "-Wl,-rpath," + libdir, "-o", exe],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    vad_dir, punc_dir = tmp_path / "vad", tmp_path / "punc"
    vad_dir.mkdir()
    punc_dir.mkdir()
    shutil.copy(vad_file, vad_dir / "vad.fab2")
    pack.write_punc_model_file(str(punc_dir / "punc.fab2"), synth.make_punc_state_dict(0), synth.PUNC_LIST, synth.punc_token_list(), 3,
                               PUNC_ENC_CONF)
    eng = SenseVoiceEngine(state, cfg, DEV, gemm_mode="fp16x3", cmvn=cmvn)
    utt = wavs[0]
    (tmp_path / "utt.wav").write_bytes(_wav_bytes(utt.numpy(), "f32"))
    long_wav = synth.make_vad_wav(*LONG_SV).numpy()
    (tmp_path / "long.wav").write_bytes(_wav_bytes(_s16(long_wav), "s16"))
    rec, vad = OfflineRecognizer(path, 0, "fp16x3"), OfflineVad(vad_file, 0)
    first = _engine_ids(eng, [utt], LID["zh"], TN["withitn"])[0]
    fired = set()
    for lang_tag in ("<|zh|>", "<|en|>"):
        # a token list that names the produced ids: the first as a language tag, the fourth as <|withitn|>, "▁" pieces elsewhere
        vocab = ["▁w%d" % i if i % 3 == 0 else "p%d" % i for i in range(cfg.vocab)]
        vocab[first[0]], vocab[first[3]] = lang_tag, "<|withitn|>"
        mdir = tmp_path / ("model_" + lang_tag[2:4])
        mdir.mkdir()
        os.symlink(path, mdir / "model.fab2")
        (mdir / "tokens.txt").write_text("\n".join(vocab) + "\n", encoding="utf-8")

        def run(audio, *extra):
            p = subprocess.run([exe, str(mdir), str(audio), *extra], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            assert p.returncode == 0, p.stdout[-2000:]
            out = dict(ln.split(" ", 1) if " " in ln else (ln, "") for ln in p.stdout.splitlines())
            assert out["asr_stamp"] == "" and out["asr_stamp_sents"] == "" and out["hotword_rows"] == "1"
            return out["asr_result"]

        for svs_lang in ("auto", "zh", "en"):
            for itn in (True, False):
                ids = _engine_ids(eng, [utt], LID[svs_lang], TN["withitn" if itn else "woitn"])[0]
                want = ctc_search_text(ids, vocab)
                assert run(tmp_path / "utt.wav", svs_lang, "1" if itn else "0") == want
                assert run(tmp_path / "utt.wav", svs_lang, "1" if itn else "0", "-", str(punc_dir)) == want
                if want.endswith("。"):
                    fired.add("zh")
                elif want.endswith("."):
                    fired.add("other")
        for svs_lang, itn in (("zh", True), ("en", False), ("klingon", True)):
            lr = rec.infer_long([_s16(long_wav)], vad, dynamic_silence=False, language=svs_lang, use_itn=itn)[0]
            want, pos = "", 0
            for k in lr["n_tokens"]:
                want += ctc_search_text(lr["token_int"][pos: pos + k], vocab)
                pos += k
            assert len(lr["n_tokens"]) >= 2
            assert run(tmp_path / "long.wav", svs_lang, "1" if itn else "0", str(vad_dir), str(punc_dir)) == want
    assert fired == {"zh", "other"}
    rec.close()
    vad.close()
