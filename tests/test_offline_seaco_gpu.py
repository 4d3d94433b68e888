"""GPU: SeacoParaformer through the C handle API.  The hotword encoder (fa_hotword_encoder_forward) against a float64 torch.nn.LSTM
restatement and the engine's cuDNN rows; the handle's ids with rows from fa_offline_hotword_embed against the reference goldens and
ParaformerEngine.forward_feats_seaco, its stamps against SeacoParaformerB200.inference, long audio against LongAudioPipeline, and the
C++ runtime surface (CompileHotwordEmbedding / FunOfflineInfer) with and without vad-dir."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT, load_seaco_case

import funasr_b200
from funasr_b200 import _abi, pack, synth
from funasr_b200.engine import FrontendEngine, ParaformerEngine, num_lfr_frames
from funasr_b200.offline import OfflineRecognizer, OfflineVad
from test_abi_host import _tiny_conf
from test_offline_vad_gpu import LONG_CASES, _vad_plugin, _wav_bytes

DEV = "cuda:0"
CFG = synth.PARAFORMER_TINY
MODES = {"fp32": 0, "fp16x3": 3}
# |row - float64 LSTM| bars per GEMM mode (rows lie in (-1, 1)); fp16x3 splits both GEMM operands into hi + lo fp16 planes.  Measured on
# an H100 80GB HBM3 at its 700 W limit: at most 2.7e-7 (fp32) and 8.4e-7 (fp16x3) over these cases, 1.9e-7 against cuDNN.
ENC_BAR = {"fp32": 1e-6, "fp16x3": 3e-6}
CUDNN_BAR = 1e-6                 # fp32 rows against the engine's cuDNN LSTM (TF32 off): two fp32 orders of the same sums


def _seaco_file(path, wseed, nfilter, cmvn=None):
    pack.write_seaco_model_file(path, synth.make_seaco_state_dict(CFG, wseed), CFG, cmvn, no_bias=synth.seaco_no_bias_id(CFG), nfilter=nfilter)
    return path


def _hotwords(n, seed, lo=1, hi=12, equal=None, outlier=None):
    g = np.random.default_rng(seed)
    out = [g.integers(3, CFG.vocab - 1, size=(equal if equal else int(g.integers(lo, hi + 1)))).tolist() for _ in range(n)]
    if outlier:
        out[n // 2] = g.integers(3, CFG.vocab - 1, size=outlier).tolist()
    return out


def _lstm64(st, hw):
    """float64 restatement of _hotword_representation: decoder.embed, the 2-layer LSTM run on each hotword alone, its last output."""
    lstm = torch.nn.LSTM(512, 512, 2, batch_first=True).double()
    lstm.load_state_dict({k[len("bias_encoder."):]: v.double() for k, v in st.items() if k.startswith("bias_encoder.")})
    emb = st["decoder.embed.0.weight"].double()
    lens = torch.tensor([len(h) for h in hw])
    pad = torch.zeros((len(hw), int(lens.max())), dtype=torch.long)
    for i, h in enumerate(hw):
        pad[i, : len(h)] = torch.tensor(h)
    with torch.no_grad():
        packed = torch.nn.utils.rnn.pack_padded_sequence(emb[pad], lens, batch_first=True, enforce_sorted=False)
        out = torch.nn.utils.rnn.pad_packed_sequence(lstm(packed)[0], batch_first=True)[0]
    return out[torch.arange(len(hw)), lens - 1].numpy()


class _Encoder:
    """fa_hotword_encoder_forward's struct over device copies of a state dict, with weight planes in the tensor-core modes."""

    def __init__(self, st, mode):
        self.lib, self.mode, self.keep = _abi.load(), MODES[mode], []
        st_ = torch.cuda.current_stream().cuda_stream

        def dev(t):
            t = t.detach().float().contiguous().to(DEV)
            self.keep.append(t)
            return t

        def lin(w, b=None):
            w = dev(w)
            b = dev(b) if b is not None else None
            planes = None
            if self.mode:
                planes = torch.empty((3, 2048, 512), dtype=torch.float16, device=DEV)
                _abi.check(self.lib.fa_split_planes(w.data_ptr(), 512, 2048, 512, 512, planes.data_ptr(), st_), "fa_split_planes")
                self.keep.append(planes)
            return _abi.FaLinear(w.data_ptr(), None if b is None else b.data_ptr(), None if planes is None else planes.data_ptr(), 2048, 512, 512, 0)

        f = lambda n, k: st["bias_encoder.%s_l%d" % (n, k)]                                         # noqa: E731
        self.ih = (_abi.FaLinear * 2)(*[lin(f("weight_ih", k), f("bias_ih", k) + f("bias_hh", k)) for k in (0, 1)])
        self.hh = (_abi.FaLinear * 2)(*[lin(f("weight_hh", k)) for k in (0, 1)])
        emb = dev(st["decoder.embed.0.weight"])
        self.enc = _abi.FaHotwordEncoder(emb.data_ptr(), CFG.vocab, 2, self.ih, self.hh)

    def __call__(self, hw):
        ids = np.array([t for h in hw for t in h], np.int32)
        lens = np.array([len(h) for h in hw], np.int32)
        ws = torch.empty(int(self.lib.fa_hotword_encoder_workspace_bytes(len(hw), ids.size, self.mode)), dtype=torch.uint8, device=DEV)
        rows = torch.full((len(hw), 512), float("nan"), device=DEV)
        _abi.check(self.lib.fa_hotword_encoder_forward(C.byref(self.enc), ids.ctypes.data, lens.ctypes.data, len(hw), rows.data_ptr(), self.mode,
                                                       ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream),
                   "fa_hotword_encoder_forward")
        torch.cuda.synchronize()
        return rows.cpu().numpy()


ENC_CASES = {"n1": dict(n=1), "n7": dict(n=7), "n25_equal": dict(n=25, equal=5), "n300_outlier": dict(n=300, outlier=40),
             "n2000": dict(n=2000)}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("case", list(ENC_CASES))
def test_hotword_encoder_vs_float64_lstm(case, mode):
    """Ragged lengths 1-12 (all equal in n25_equal, one 40-token outlier in n300_outlier): every row within the mode's bar of the float64
    LSTM, and in fp32 within fp32 noise of the engine's cuDNN rows.  Each hotword alone gives its batch row bit for bit."""
    st = synth.make_seaco_state_dict(CFG, 10)
    hw = _hotwords(seed=len(case) * 31 + ENC_CASES[case]["n"], **ENC_CASES[case])
    enc = _Encoder(st, mode)
    rows = enc(hw)
    ref = _lstm64(st, hw)
    err = float(np.abs(rows - ref).max())
    print("hotword encoder %s %s: max |row - float64| %.3e" % (case, mode, err))
    assert np.isfinite(rows).all() and err <= ENC_BAR[mode], err
    if mode == "fp32":
        eng = ParaformerEngine(st, CFG, DEV, gemm_mode="fp32", seaco=True, no_bias=synth.seaco_no_bias_id(CFG))
        cud = eng.seaco_hotword_representation(hw).cpu().numpy()
        print("hotword encoder %s: max |row - cuDNN| %.3e" % (case, float(np.abs(rows - cud).max())))
        assert float(np.abs(rows - cud).max()) <= CUDNN_BAR
    for i in (0, len(hw) - 1):
        assert np.array_equal(enc([hw[i]])[0], rows[i])


@pytest.mark.gpu
def test_hotword_encoder_refusals_on_the_device():
    """Out-of-vocabulary ids, n = 0 and NULL pointers are refused before any launch; a real call after them still works."""
    lib = _abi.load()
    st = synth.make_seaco_state_dict(CFG, 10)
    enc = _Encoder(st, "fp16x3")
    hw = _hotwords(5, 3)
    ids = np.array([t for h in hw for t in h], np.int32)
    lens = np.array([len(h) for h in hw], np.int32)
    ws = torch.empty(int(lib.fa_hotword_encoder_workspace_bytes(5, ids.size, 3)), dtype=torch.uint8, device=DEV)
    rows = torch.zeros((5, 512), device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    call = lambda i, ln, n, r: lib.fa_hotword_encoder_forward(C.byref(enc.enc), i, ln, n, r, 3, ws.data_ptr(), ws.numel(), s)   # noqa: E731
    l0 = lib.fa_launch_count()
    bad = ids.copy()
    bad[-1] = CFG.vocab
    assert call(bad.ctypes.data, lens.ctypes.data, 5, rows.data_ptr()) == -1
    assert call(ids.ctypes.data, lens.ctypes.data, 0, rows.data_ptr()) == -1
    assert call(None, lens.ctypes.data, 5, rows.data_ptr()) == -1 and call(ids.ctypes.data, lens.ctypes.data, 5, None) == -1
    assert lib.fa_launch_count() == l0
    assert float(rows.abs().max()) == 0.0
    assert call(ids.ctypes.data, lens.ctypes.data, 5, rows.data_ptr()) == 0
    torch.cuda.synchronize()
    assert np.array_equal(rows.cpu().numpy(), enc(hw))


def _engine_ids(st, mode, wavs, cmvn, hw, nfilter):
    eng = ParaformerEngine(st, CFG, DEV, gemm_mode=mode, seaco=True, no_bias=synth.seaco_no_bias_id(CFG))
    fe = FrontendEngine(cmvn, DEV)
    lens = [w.numel() for w in wavs]
    pad = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True).to(DEV)
    feats, fl = fe(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), max(num_lfr_frames(n) for n in lens))
    return eng.forward_feats_seaco(feats, fl, hw, nfilter=nfilter)["ids"], eng.forward_feats_seaco(feats, fl, None)["ids"]


def _plugin(st, mode, cmvn):
    conf = _tiny_conf()
    conf["gemm_mode"] = mode
    conf["predictor"] = "CifPredictorV3B200"
    conf["predictor_conf"] = dict(idim=512, threshold=1.0, l_order=1, r_order=1, tail_threshold=CFG.tail_threshold, smooth_factor2=0.25,
                                  noise_threshold2=0.01, upsample_times=3, use_cif1_cnn=False, upsample_type="cnn_blstm")
    m = funasr_b200.SeacoParaformerB200(**conf, seaco_decoder="ParaformerSANMDecoder", inner_dim=512, NO_BIAS=synth.seaco_no_bias_id(CFG),
                                        seaco_decoder_conf=dict(attention_heads=4, linear_units=synth.SEACO_FFN, num_blocks=4,
                                                                kernel_size=synth.SEACO_KERNEL, sanm_shfit=0, use_output_layer=False,
                                                                wo_input_layer=True))
    m.load_state_dict(st, strict=True)
    m.to(DEV).eval()
    fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0, cmvn=cmvn)
    return m, fe


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
@pytest.mark.parametrize("name", ["seaco_tiny_ragged3", "seaco_tiny_asf"])
def test_handle_ids_vs_reference_golden_engine_and_plugin(tmp_path, name, mode):
    """Rows from fa_offline_hotword_embed for the fixture's hotword list: the handle's ids equal the unmodified reference's goldens (the
    second case runs the attention-score filter: 24 hotwords + <s>, nfilter 8) and forward_feats_seaco; without rows they equal
    forward_feats_seaco(hw_list=None); the stamps equal SeacoParaformerB200.inference's."""
    cfg, wseed, wavs, cmvn, hw, nfilter, g = load_seaco_case(name)
    assert cfg is CFG
    st = synth.make_seaco_state_dict(CFG, wseed)
    rec = OfflineRecognizer(_seaco_file(str(tmp_path / "m.fab2"), wseed, nfilter, cmvn), 0, mode)
    assert rec.is_seaco and rec.has_timestamps and not rec.is_sensevoice
    rows = rec.hotword_embeddings(hw)
    assert rows.shape == (len(hw), 512)
    if name == "seaco_tiny_asf":
        assert len(hw) > nfilter
    got = rec.infer_stamped([w.numpy() for w in wavs], hotword_embeddings=rows)
    ids = [r["token_int"] for r in got]
    assert [t for r in ids for t in r] == g["ids_flat"].tolist() and [len(r) for r in ids] == g["ids_len"].tolist()
    want, want_plain = _engine_ids(st, mode, wavs, cmvn, hw, nfilter)
    assert ids == want
    assert rec.infer([w.numpy() for w in wavs]) == want_plain
    m, fe = _plugin(st, mode, cmvn)
    res, _ = m.inference([w.numpy() for w in wavs], key=["a%d" % i for i in range(len(wavs))], tokenizer=None, frontend=fe, device=DEV,
                         hotword_ids=hw, nfilter=nfilter)
    assert [r["token_int"] for r in res] == ids
    assert [r["timestamp"] for r in res] == [r["timestamp"] for r in got]
    rec.close()


@pytest.fixture(scope="module")
def vad_file(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("vad") / "vad.fab2")
    pack.write_vad_model_file(path, synth.make_vad_state_dict(synth.VAD_DEFAULT, 0), synth.make_vad_cmvn(0), {})
    return path


LONG_SEED, LONG_NFILTER = 11, 8


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "fp16x3"])
def test_long_audio_with_hotwords_vs_pipeline(tmp_path, vad_file, mode):
    """fa_offline_infer_vad with SeACo rows on the 40 s recording in 6 s packs (several packs, the filter on each pack's first segment:
    24 hotwords + <s>, nfilter 8) equals LongAudioPipeline over SeacoParaformerB200 with hotword_ids; three recordings in one call equal
    three calls."""
    cmvn = synth.make_cmvn(CFG, 1)
    st = synth.make_seaco_state_dict(CFG, LONG_SEED)
    rec, vad = OfflineRecognizer(_seaco_file(str(tmp_path / "m.fab2"), LONG_SEED, LONG_NFILTER, cmvn), 0, mode), OfflineVad(vad_file, 0)
    hw = synth.make_hotwords(24, CFG.vocab, seed=9)
    rows = rec.hotword_embeddings(hw)
    wavs = [synth.make_vad_wav(*LONG_CASES[k][:3]).numpy() for k in ("longaudio_40s", "longaudio_25s_onebatch")]
    wavs.append(wavs[0][: 16000 * 17].copy())
    got = rec.infer_long(wavs, vad, batch_size_s=6, hotword_embeddings=rows)
    assert len(got[0]["vad_segments"]) >= 2 and got[0]["token_int"] and got[0]["timestamp"]
    m, fe = _plugin(st, mode, cmvn)
    v, v_fe = _vad_plugin()
    pipe = funasr_b200.LongAudioPipeline(m, fe, v, v_fe, device=DEV, tokenizer=None)
    want = pipe.generate(wavs[0], key="rec", batch_size_s=6, hotword_ids=hw, nfilter=LONG_NFILTER)
    assert got[0]["token_int"] == want["token_int"] and got[0]["timestamp"] == want["timestamp"]
    assert got[0]["vad_segments"] == want["vad_segments"]
    for i, w in enumerate(wavs):
        assert rec.infer_long([w], vad, batch_size_s=6, hotword_embeddings=rows)[0] == got[i], i
    plain = rec.infer_long(wavs[:1], vad, batch_size_s=6)[0]
    assert plain["token_int"] == pipe.generate(wavs[0], key="rec", batch_size_s=6)["token_int"]
    rec.close()
    vad.close()


CLIENT = r'''
#include <stdio.h>
#include "funasrruntime_b200.h"
int main(int argc, char** argv) {
  std::map<std::string, std::string> mp;
  mp["model-dir"] = argv[1];
  mp["gemm-mode"] = "fp16x3";
  if (argc > 5) mp["vad-dir"] = argv[5];
  FUNASR_HANDLE h = FunOfflineInit(mp, 1);
  if (!h) { printf("init failed %s\n", FunB200LastError()); return 1; }
  std::string words = argv[3];
  std::vector<std::vector<float>> hw = CompileHotwordEmbedding(h, words);
  FILE* f = fopen(argv[4], "wb");
  for (const auto& r : hw) fwrite(r.data(), 4, r.size(), f);
  fclose(f);
  FUNASR_RESULT r = FunOfflineInfer(h, argv[2], RASR_NONE, nullptr, hw, 16000);
  if (!r) { printf("infer failed %s\n", FunB200LastError()); return 1; }
  printf("rows %zu\ntext %s\nstamp %s\n", hw.size(), FunASRGetResult(r, 0), FunASRGetStamp(r));
  FunASRFreeResult(r);
  FunOfflineUninit(h);
  return 0;
}
'''


@pytest.mark.gpu
def test_runtime_client_with_hotwords(tmp_path, vad_file):
    """A SeACo model-dir with tokens.txt: examples/offline_runtime_client.cpp, built unchanged, prints the text of the handle's ids for
    a hotword string; a client of the same surface with vad-dir too.  CompileHotwordEmbedding's rows equal fa_offline_hotword_embed for
    the parsed ids (an out-of-vocabulary hotword dropped, <s> appended)."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    _, wseed, wavs, cmvn, hw, nfilter, _ = load_seaco_case("seaco_tiny_asf")
    d, vd = tmp_path / "asr", tmp_path / "vad"
    d.mkdir()
    vd.mkdir()
    model = _seaco_file(str(d / "model.fab2"), wseed, nfilter, cmvn)
    os.symlink(vad_file, str(vd / "vad.fab2"))
    tokens = ["<blank>", "<s>", "</s>"] + [chr(0x4E00 + i) for i in range(3, CFG.vocab)]
    (d / "tokens.txt").write_text("\n".join(tokens) + "\n", encoding="utf-8")
    words = " ".join("".join(tokens[t] for t in h) for h in hw[:-1]) + " あ"        # the last one is not in tokens.txt
    inc, libdir = os.path.join(ROOT, "include"), os.path.join(ROOT, "funasr_b200")
    exe_ex, exe = str(tmp_path / "example"), str(tmp_path / "client")
    (tmp_path / "client.cpp").write_text(CLIENT)
    for src, out in ((os.path.join(ROOT, "examples", "offline_runtime_client.cpp"), exe_ex), (str(tmp_path / "client.cpp"), exe)):
        r = subprocess.run(["g++", "-std=c++17", "-I" + inc, src, "-L" + libdir, "-lfunasr_b200", "-Wl,-rpath," + libdir, "-o", out],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout[-2000:]
    rec, vad = OfflineRecognizer(model, 0, "fp16x3"), OfflineVad(vad_file, 0)
    rows = rec.hotword_embeddings(hw)
    text = lambda ids: "".join(tokens[t] for t in ids)                                   # noqa: E731
    short = wavs[0].numpy()
    wav_path = str(tmp_path / "short.wav")
    open(wav_path, "wb").write(_wav_bytes(short, "f32"))
    want = text(rec.infer([short], hotword_embeddings=rows)[0])
    p = subprocess.run([exe_ex, str(d), wav_path, "fp16x3", words], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-2000:]
    out = dict(ln.split(" ", 1) for ln in p.stdout.splitlines() if " " in ln)
    assert out["hotword_rows"] == str(len(hw)) and out["file_result"] == want and out["buffer_result"] == want
    p = subprocess.run([exe, str(d), wav_path, words, str(tmp_path / "rows.bin")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-2000:]
    assert np.array_equal(np.fromfile(str(tmp_path / "rows.bin"), np.float32).reshape(-1, 512), rows)
    long = synth.make_vad_wav(*LONG_CASES["longaudio_40s"][:3]).numpy()
    long_path = str(tmp_path / "long.wav")
    open(long_path, "wb").write(_wav_bytes(long, "f32"))
    p = subprocess.run([exe, str(d), long_path, words, str(tmp_path / "rows2.bin"), str(vd)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True)
    assert p.returncode == 0, p.stdout[-2000:]
    out = dict(ln.split(" ", 1) if " " in ln else (ln, "") for ln in p.stdout.splitlines())
    got = rec.infer_long([long], vad, hotword_embeddings=rows, dynamic_silence=False)[0]
    assert out["text"] == text(got["token_int"]) and got["token_int"]
    assert out["stamp"] == "[" + ",".join("[%d,%d]" % (a, b) for a, b in got["timestamp"]) + "]"
    rec.close()
    vad.close()
