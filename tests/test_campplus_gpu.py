"""CAM++ speaker embeddings and diarization on the GPU: every kernel against a float64 CPU restatement of its layer, features and
embeddings against the reference's stored results, and the whole LongAudioPipeline(spk_model=...) against the reference's labels and
sentence_info.  Fixtures: oracle/make_spk_golden.py."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from campplus_ref import cam_layer_ref, campplus_ref
from test_spk_host import SPK_CASES, campplus_state_dict, load_spk_case

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MODES = ["fp32", "fp16x3"]


def _st():
    return torch.cuda.current_stream(DEV).cuda_stream


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


# ---------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("cin,k,stride,f_in,t,res,relu", [(1, 3, 1, 80, 148, False, True), (32, 3, 2, 80, 37, False, True),
                                                           (32, 3, 1, 40, 61, True, True), (32, 1, 2, 40, 29, False, False),
                                                           (32, 3, 2, 20, 5, False, True),
                                                           # a partial kConvTP = 4 time tile only
                                                           (1, 3, 1, 80, 1, False, True), (32, 3, 1, 40, 2, True, True),
                                                           (32, 3, 2, 20, 3, False, True)])
def test_fcm_conv_kernel(cin, k, stride, f_in, t, res, relu):
    from funasr_b200 import _abi
    lib = _abi.load()
    g = torch.Generator().manual_seed(cin * 100 + k * 10 + stride + t)
    B = 3
    x = torch.randn(B, cin, f_in, t, generator=g)
    w = torch.randn(32, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(32, generator=g) * 0.1
    ref = F.conv2d(x.double(), w.double(), b.double(), stride=(stride, 1), padding=k // 2)
    r = torch.randn_like(ref) if res else None
    if res:
        ref = ref + r
    if relu:
        ref = F.relu(ref)
    xd = x.permute(0, 2, 3, 1).contiguous().to(DEV)                           # channels last [B][F][T][C]
    wd = w.permute(2, 3, 1, 0).reshape(k * k, cin, 32).contiguous().to(DEV)
    bd = b.to(DEV)
    f_out = ref.shape[2]
    y = torch.empty(B, f_out, t, 32, device=DEV)
    rd = r.float().permute(0, 2, 3, 1).contiguous().to(DEV) if res else None
    conv = _abi.FaCamConv2d(wd.data_ptr(), bd.data_ptr(), cin, 32, k, stride)
    _abi.check(lib.fa_campplus_conv2d(C.byref(conv), xd.data_ptr(), B, f_in, t, None if rd is None else rd.data_ptr(), y.data_ptr(),
                                      int(relu), _st()), "fa_campplus_conv2d")
    assert rel(y.permute(0, 3, 1, 2), ref) < 1e-5


# t 100 / 101 / 199: one full segment, a one-row last segment, a 99-row last segment; dil 8 is kCamMaxDil; t 9 400 is the most segments
# (94) the gate kernel's shared memory holds.  dil 9 and t 9 401 are refused before any launch.
@pytest.mark.parametrize("t,dil", [(74, 1), (74, 2), (150, 2), (201, 1), (1, 2), (100, 2), (101, 2), (199, 2), (74, 8), (9400, 2),
                                   (74, 9), (9401, 2)])
def test_cam_kernel(t, dil):
    from funasr_b200 import _abi
    lib = _abi.load()
    if dil > 8 or t > 9400:
        B = 2
        h = torch.zeros(B * t, 128, device=DEV)
        w = torch.zeros(3 * 128 * 32, device=DEV)
        gates = torch.empty(B, (t + 99) // 100, 32, device=DEV)
        out = torch.empty(B * t, 32, device=DEV)
        torch.cuda.synchronize()
        n0 = lib.fa_launch_count()
        rc = lib.fa_campplus_cam(h.data_ptr(), B, t, dil, *([w.data_ptr()] * 5), gates.data_ptr(), out.data_ptr(), 32, _st())
        torch.cuda.synchronize()
        assert rc == (-1 if dil > 8 else -4) and lib.fa_launch_count() == n0
        return
    g = torch.Generator().manual_seed(t * 10 + dil)
    B = 5
    h = F.relu(torch.randn(B, 128, t, generator=g))
    wl = torch.randn(32, 128, 3, generator=g) / 20
    w1, b1 = torch.randn(64, 128, 1, generator=g) / 11, torch.randn(64, generator=g) * 0.1
    w2, b2 = torch.randn(32, 64, 1, generator=g) / 8, torch.randn(32, generator=g) * 0.1
    ref = cam_layer_ref(h.double(), wl.double(), w1.double(), b1.double(), w2.double(), b2.double(), dil)
    hd = h.permute(0, 2, 1).contiguous().to(DEV)
    dev = [u.contiguous().to(DEV) for u in (wl.permute(2, 1, 0), w1[:, :, 0], b1, w2[:, :, 0], b2)]
    nseg = (t + 99) // 100
    gates = torch.empty(B, nseg, 32, device=DEV)
    ld = 96
    out = torch.full((B * t, ld), 7.0, device=DEV)
    _abi.check(lib.fa_campplus_cam(hd.data_ptr(), B, t, dil, *[u.data_ptr() for u in dev], gates.data_ptr(), out[:, 32:].data_ptr(), ld, _st()),
               "fa_campplus_cam")
    got = out[:, 32:64].reshape(B, t, 32).permute(0, 2, 1)
    print("campplus cam t%d dil%d: rel %.3e" % (t, dil, rel(got, ref)))
    assert rel(got, ref) < 1e-5
    assert bool((out[:, :32] == 7.0).all()) and bool((out[:, 64:] == 7.0).all())        # only its column slice is written


# t 1: the mean is y itself and the unbiased std 0 / 0 (NaN, as torch.std(unbiased=True) gives); t 9 400: the longest fp32 time sum
@pytest.mark.parametrize("t", [74, 3, 257, 1, 2, 9400])
def test_stats_pool_kernel(t):
    from funasr_b200 import _abi
    lib = _abi.load()
    g = torch.Generator().manual_seed(t)
    B, Cc = 4, 512
    x = torch.randn(B, t, Cc, generator=g)
    s, sh = 1.0 + 0.2 * torch.randn(Cc, generator=g), 0.3 * torch.randn(Cc, generator=g)
    y = F.relu(x.double() * s.double() + sh.double())
    ref = torch.cat([y.mean(1), y.std(1, unbiased=True)], -1)
    xd, sd_, shd = x.to(DEV), s.to(DEV), sh.to(DEV)
    out = torch.empty(B, 2 * Cc, device=DEV)
    _abi.check(lib.fa_campplus_stats_pool(xd.data_ptr(), B, t, Cc, sd_.data_ptr(), shd.data_ptr(), out.data_ptr(), _st()), "fa_campplus_stats_pool")
    if t == 1:
        assert torch.equal(out[:, :Cc].cpu(), y[:, 0].float())          # fmaf rounds x * s + sh once, like float64 then fp32
        assert bool(torch.isnan(out[:, Cc:]).all()) and bool(torch.isnan(ref[:, Cc:]).all())
        return
    print("campplus stats t%d: rel %.3e" % (t, rel(out, ref)))
    # the time sums run in fp32 in time order, so their rounding grows with t: 2.8e-5 at t 9 400 on an H100 (8.7e-7 at t 257)
    assert rel(out, ref) < (1.2e-4 if t > 1000 else 1e-5)


# ---------------------------------------------------------------------------------------------- model level
def _engine(mode):
    from funasr_b200.campplus import CampplusEngine
    return CampplusEngine(campplus_state_dict(), DEV, mode)


def _chunk_batch(name):
    from funasr_b200 import synth
    from funasr_b200.long_audio import speaker_chunks
    from test_spk_host import vad_segments
    pattern, seed, _ = SPK_CASES[name]
    g = load_spk_case(name)
    wav = synth.make_voice_wav(pattern, seed)
    ch = speaker_chunks(vad_segments(g), wav.numel())
    batch = torch.zeros(len(ch), 24000)
    for i, (_, _, s, n) in enumerate(ch):
        batch[i, :n] = wav[s:s + n]
    return g, batch


@pytest.mark.parametrize("name", list(SPK_CASES))
def test_features_vs_reference(name):
    g, batch = _chunk_batch(name)
    eng = _engine("fp32")
    feats, flens = eng.features(batch[:4].contiguous().to(DEV), torch.full((4,), 24000, dtype=torch.int32, device=DEV), 148)
    assert flens.tolist() == [148] * 4
    assert float((feats.cpu() - torch.from_numpy(g["features"])).abs().max()) < 1e-4


@pytest.mark.parametrize("mode", MODES)
def test_embeddings_vs_reference(mode):
    """Embeddings of every fixture chunk, from the waveform, against the reference CAMPPlus (stored).  The float64 parity of the
    forward in every mode is test_campplus_entries_gpu.py's."""
    eng = _engine(mode)
    errs = []
    for name in SPK_CASES:
        g, batch = _chunk_batch(name)
        n = batch.shape[0]
        emb = eng.embed_wav(batch.to(DEV), torch.full((n,), 24000, dtype=torch.int32, device=DEV), [24000] * n)
        errs.append(rel(emb, g["cb_in"]))
    print("CAM++ %s embeddings: max rel err vs reference %.2e" % (mode, max(errs)))
    assert max(errs) < 1e-3


@pytest.mark.parametrize("mode", MODES)
def test_malformed_last_layer_launches_nothing(mode):
    """A malformed last dense layer or last transit is refused (-1) before the first launch: fa_launch_count() is unchanged."""
    from funasr_b200 import _abi
    eng = _engine(mode)
    lib = eng.lib
    n = sum(eng.model.n_layers)
    B, T = 2, 148
    feats = torch.randn(B, T, 80, device=DEV)
    emb = torch.empty(B, eng.model.dense.out_f, device=DEV)

    def run(m):
        ws = torch.empty(int(lib.fa_campplus_workspace_bytes(C.byref(m), B, T, eng.mode)), dtype=torch.uint8, device=DEV)
        torch.cuda.synchronize()
        n0 = lib.fa_launch_count()
        rc = lib.fa_campplus_forward(C.byref(m), feats.data_ptr(), B, T, emb.data_ptr(), eng.mode, ws.data_ptr(), ws.numel(), _st())
        torch.cuda.synchronize()
        return rc, int(lib.fa_launch_count() - n0)

    rc, launched = run(eng.model)
    assert rc == 0 and launched > 0
    for fault in ("layer", "transit"):
        layers = (_abi.FaCamLayer * n)()
        for i in range(n):
            layers[i] = _abi.FaCamLayer.from_buffer_copy(eng.layers[i])
        m = _abi.FaCampplus.from_buffer_copy(eng.model)
        m.layers = layers
        if fault == "layer":
            layers[n - 1].linear1.in_f += 32
        else:
            m.transit[2].linear.in_f += 1
        assert run(m) == (-1, 0)


def test_inference_contract_ragged():
    """CAMPPlusB200.inference: a list of ragged waveforms -> [{"spk_embedding": [B, 192]}], features zero-padded to the longest input
    (pad_list) and every padded frame taking part, batch_data_time in seconds."""
    from funasr_b200 import synth
    from funasr_b200.campplus import CAMPPlusB200
    m = CAMPPlusB200()
    m.load_state_dict(campplus_state_dict(), strict=True)
    wavs = [synth.make_voice_wav([(0, 1.2, 0.1)], 5), synth.make_voice_wav([(1, 2.3, 0.1)], 6).numpy(), synth.make_voice_wav([(2, 0.6, 0.1)], 7)]
    res, meta = m.inference(wavs, device=DEV)
    emb = res[0]["spk_embedding"]
    assert tuple(emb.shape) == (3, 192) and emb.is_cuda
    lens = [int(np.asarray(w).size) for w in wavs]
    assert abs(meta["batch_data_time"] - sum(lens) / 16000.0) < 1e-9
    # the same padded features through the float64 restatement
    eng = m.engine(DEV)
    pad = torch.nn.utils.rnn.pad_sequence([torch.as_tensor(w).float() for w in wavs], batch_first=True).to(DEV)
    t_max = max(1 + (n - 400) // 160 for n in lens)
    feats, flens = eng.features(pad, torch.tensor(lens, dtype=torch.int32, device=DEV), t_max)
    assert flens.tolist() == [1 + (n - 400) // 160 for n in lens]
    assert float(feats[2, flens[2]:].abs().max()) == 0.0
    ref = campplus_ref(campplus_state_dict(), feats.cpu())
    assert rel(emb, ref) < 1e-3
    # one input alone gives a different embedding than inside the padded batch (the reference's unmasked means)
    alone = m.inference([wavs[2]], device=DEV)[0][0]["spk_embedding"]
    assert rel(alone[0], emb[2]) > 1e-3


# ---------------------------------------------------------------------------------------------- pipeline
def _pipeline(mode):
    import funasr_b200
    from funasr_b200 import synth
    from test_abi_host import _tiny_conf
    cfg = synth.PARAFORMER_TINY
    asr = funasr_b200.ParaformerB200(**_tiny_conf())
    asr.load_state_dict(synth.make_state_dict(cfg, 3), strict=True)
    asr.to(DEV).eval()
    asr_fe = funasr_b200.WavFrontendB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=7, lfr_n=6, dither=0.0,
                                         cmvn=synth.make_cmvn(cfg, 1))
    c = synth.VAD_DEFAULT
    vad = funasr_b200.FsmnVADStreamingB200(encoder="FSMN", encoder_conf=dict(
        input_dim=c.input_dim, input_affine_dim=c.input_affine_dim, fsmn_layers=c.fsmn_layers, linear_dim=c.linear_dim, proj_dim=c.proj_dim,
        lorder=c.lorder, rorder=0, lstride=1, rstride=0, output_affine_dim=c.output_affine_dim, output_dim=c.output_dim))
    vad.load_state_dict(synth.make_vad_state_dict(c, 0), strict=True)
    vad.to(DEV).eval()
    vad_fe = funasr_b200.WavFrontendOnlineB200(fs=16000, window="hamming", n_mels=80, frame_length=25, frame_shift=10, lfr_m=5, lfr_n=1,
                                               dither=0.0, cmvn=synth.make_vad_cmvn(0))
    spk = funasr_b200.CAMPPlusB200(gemm_mode=mode)
    spk.load_state_dict(campplus_state_dict(), strict=True)
    return funasr_b200.LongAudioPipeline(asr, asr_fe, vad, vad_fe, device=DEV, spk_model=spk), (asr, asr_fe, vad, vad_fe)


@pytest.mark.parametrize("mode", MODES)
def test_pipeline_diarization_vs_reference(mode):
    """LongAudioPipeline(spk_model=CAMPPlusB200) on every fixture: VAD segments, chunk labels and sentence_info speakers identical to the
    reference AutoModel(..., spk_model="CAMPPlus") in vad_segment mode; sentence timestamps absolute; spk_embedding_center when asked."""
    from funasr_b200 import diarization as D
    from funasr_b200 import synth
    pipe, _ = _pipeline(mode)
    for name, (pattern, seed, kw) in SPK_CASES.items():
        g = load_spk_case(name)
        wav = synth.make_voice_wav(pattern, seed)
        out = pipe.generate(wav.numpy(), key="rec", pred_timestamp=True, batch_size_s=300, **kw)
        info = out["sentence_info"]
        assert [[s["start"], s["end"]] for s in info] == g["segments"].tolist(), name
        assert [s["spk"] for s in info] == [s["spk"] for s in g["sentence_info"]], name
        labels = D.ClusterBackend()(out["spk_embedding"].cpu().numpy(), oracle_num=kw.get("preset_spk_num"))
        assert D.correct_labels(labels).tolist() == D.correct_labels(g["labels"]).tolist(), name
        for s in info:
            assert all(s["start"] <= a <= b for a, b in s["timestamp"])
        if kw.get("return_spk_center"):
            assert out["spk_embedding_center"].shape == g["spk_embedding_center"].shape
            assert rel(out["spk_embedding_center"], g["spk_embedding_center"]) < 1e-3


def test_pipeline_without_spk_model_unchanged():
    """No speaker model: the result carries no speaker keys and equals the pipeline built without the argument."""
    import funasr_b200
    from funasr_b200 import synth
    pipe, parts = _pipeline("fp32")
    plain = funasr_b200.LongAudioPipeline(*parts, device=DEV)
    wav = synth.make_voice_wav(SPK_CASES["spk_few_chunks"][0], 3).numpy()
    a = plain.generate(wav, key="rec", pred_timestamp=True)
    assert not any(k in a for k in ("sentence_info", "spk_embedding"))
    b = funasr_b200.LongAudioPipeline(*parts, device=DEV, spk_model=None).generate(wav, key="rec", pred_timestamp=True)
    assert a == b
