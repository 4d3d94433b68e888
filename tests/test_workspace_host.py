"""The *_workspace_bytes queries are host code: each is the measuring run of the carve its forward uses.  Their values are pinned
here over the shapes the project runs, in every GEMM mode, next to what the queries returned before they shared the forward's
carve: no query may grow, and where a path keeps every buffer (fp32) only alignment padding and headroom went away."""
import ctypes as C

import pytest

from funasr_b200 import _abi

MODES = {"fp32": _abi.GEMM_F32_SIMT, "fp16": _abi.GEMM_F16X1, "fp16x3": _abi.GEMM_F16X3, "fp16x6": _abi.GEMM_F16X6}


def _vad():
    """FSMN-VAD widths: in_linear1 -> 140, in_linear2 -> 250, out_linear1 -> 140, out_linear2 -> 248 classes."""
    e = _abi.FaVadEncoder()
    e.in1.out_f, e.in2.out_f, e.out1.out_f, e.out2.out_f = 140, 250, 140, 248
    return e


def _cam():
    """CAM++ (speech_campplus_sv_zh-cn_16k-common): dense blocks of 12, 24 and 16 layers."""
    m = _abi.FaCampplus()
    m.n_layers[0], m.n_layers[1], m.n_layers[2] = 12, 24, 16
    return m


# (query, shape, arguments with "m" standing for the GEMM mode): tiny, bench config 2 (64 x 500 LFR frames, 128 tokens, 33
# hotwords), bench config 4 (64 x 504 frames, 25055-entry CTC vocabulary), the fa-zh aligner, punctuation, VAD and CAM++
CASES = [
    ("fa_sanm_encoder_workspace_bytes", "tiny", (3, 37, "m")),
    ("fa_sanm_encoder_workspace_bytes", "config2", (64, 500, "m")),
    ("fa_sanm_encoder_workspace_bytes", "config4", (64, 504, "m")),
    ("fa_sanm_encoder_workspace_bytes", "aligner", (8, 300, "m")),
    ("fa_sanm_encoder_workspace_bytes", "punc", (1, 200, "m")),
    ("fa_cif_predictor_workspace_bytes", "tiny", (3, 37, "m")),
    ("fa_cif_predictor_workspace_bytes", "config2", (64, 500, "m")),
    ("fa_paraformer_decoder_workspace_bytes_hw", "tiny", (3, 37, 9, 8404, "m", 0)),
    ("fa_paraformer_decoder_workspace_bytes_hw", "tiny_hotwords", (3, 37, 9, 8404, "m", 5)),
    ("fa_paraformer_decoder_workspace_bytes_hw", "config2", (64, 500, 128, 8404, "m", 0)),
    ("fa_paraformer_decoder_workspace_bytes_hw", "config2_hotwords", (64, 500, 128, 8404, "m", 33)),
    ("fa_sanm_decoder_stack_workspace_bytes", "tiny", (3, 5, 9, "m")),
    ("fa_sanm_decoder_stack_workspace_bytes", "config2", (64, 33, 128, "m")),
    ("fa_linear_argmax_workspace_bytes", "tiny", (27, 8404, "m")),
    ("fa_linear_argmax_workspace_bytes", "config2", (64 * 128, 8404, "m")),
    ("fa_linear_argmax_workspace_bytes", "punc", (200, 6, "m")),
    ("fa_ctc_greedy_workspace_bytes", "tiny", (3, 37, 25055, "m")),
    ("fa_ctc_greedy_workspace_bytes", "config4", (64, 504, 25055, "m")),
    ("fa_attention_tc_workspace_bytes", "tiny", (3, 4, 9, 37, "m")),
    ("fa_attention_tc_workspace_bytes", "config2", (64, 4, 500, 500, "m")),
    ("fa_campplus_workspace_bytes", "tiny", ("cam", 1, 148, "m")),
    ("fa_campplus_workspace_bytes", "spk", ("cam", 16, 300, "m")),
    ("fa_fsmn_vad_workspace_bytes", "vad_30s", ("vad", 3000)),
    ("fa_fsmn_vad_workspace_bytes", "vad_130s", ("vad", 13000)),
    ("fa_blstm_tc_scratch_bytes", "tiny", (3,)),
    ("fa_blstm_tc_scratch_bytes", "aligner", (8,)),
    ("fa_blstm_tc_scratch_bytes", "max", (256,)),
    ("fa_timestamp_head_workspace_bytes", "tiny", (3, 37, 512, 3, "m")),
    ("fa_timestamp_head_workspace_bytes", "config2", (64, 500, 512, 3, "m")),
    ("fa_timestamp_head_workspace_bytes", "aligner", (8, 300, 320, 3, "m")),
]

# (query, shape, mode) -> (value before the queries ran the forward's carve, value now)
VALUES = {
    ("fa_sanm_encoder_workspace_bytes", "tiny", "fp32"): (2749696, 2749440),
    ("fa_sanm_encoder_workspace_bytes", "tiny", "fp16"): (6141952, 2484224),
    ("fa_sanm_encoder_workspace_bytes", "tiny", "fp16x3"): (6596608, 3604224),
    ("fa_sanm_encoder_workspace_bytes", "tiny", "fp16x6"): (7051264, 4300544),
    ("fa_sanm_encoder_workspace_bytes", "config2", "fp32"): (792576256, 792576000),
    ("fa_sanm_encoder_workspace_bytes", "config2", "fp16"): (1723942144, 693010432),
    ("fa_sanm_encoder_workspace_bytes", "config2", "fp16x3"): (1855014144, 992804864),
    ("fa_sanm_encoder_workspace_bytes", "config2", "fp16x6"): (1986086144, 1193508864),
    ("fa_sanm_encoder_workspace_bytes", "config4", "fp32"): (798916864, 798916608),
    ("fa_sanm_encoder_workspace_bytes", "config4", "fp16"): (1737196800, 698286080),
    ("fa_sanm_encoder_workspace_bytes", "config4", "fp16x3"): (1869317376, 1000210432),
    ("fa_sanm_encoder_workspace_bytes", "config4", "fp16x6"): (2001437952, 1202520064),
    ("fa_sanm_encoder_workspace_bytes", "aligner", "fp32"): (59443456, 59443200),
    ("fa_sanm_encoder_workspace_bytes", "aligner", "fp16"): (129506560, 52080640),
    ("fa_sanm_encoder_workspace_bytes", "aligner", "fp16x3"): (139336960, 74670080),
    ("fa_sanm_encoder_workspace_bytes", "aligner", "fp16x6"): (149167360, 89722880),
    ("fa_sanm_encoder_workspace_bytes", "punc", "fp32"): (4953856, 4953600),
    ("fa_sanm_encoder_workspace_bytes", "punc", "fp16"): (10880768, 4383744),
    ("fa_sanm_encoder_workspace_bytes", "punc", "fp16x3"): (11699968, 6309888),
    ("fa_sanm_encoder_workspace_bytes", "punc", "fp16x6"): (12519168, 7564288),
    ("fa_cif_predictor_workspace_bytes", "tiny", "fp32"): (910080, 909756),
    ("fa_cif_predictor_workspace_bytes", "tiny", "fp16"): (1252096, 361984),
    ("fa_cif_predictor_workspace_bytes", "tiny", "fp16x3"): (1593088, 483840),
    ("fa_cif_predictor_workspace_bytes", "tiny", "fp16x6"): (1934080, 605696),
    ("fa_cif_predictor_workspace_bytes", "config2", "fp32"): (262272256, 262272000),
    ("fa_cif_predictor_workspace_bytes", "config2", "fp16"): (360577280, 98827264),
    ("fa_cif_predictor_workspace_bytes", "config2", "fp16x3"): (458881280, 131728384),
    ("fa_cif_predictor_workspace_bytes", "config2", "fp16x6"): (557185280, 164629504),
    ("fa_paraformer_decoder_workspace_bytes_hw", "tiny", "fp32"): (2026240, 1915248),
    ("fa_paraformer_decoder_workspace_bytes_hw", "tiny", "fp16"): (3996416, 1967616),
    ("fa_paraformer_decoder_workspace_bytes_hw", "tiny", "fp16x3"): (4451072, 2585088),
    ("fa_paraformer_decoder_workspace_bytes_hw", "tiny", "fp16x6"): (4905728, 2864640),
    ("fa_paraformer_decoder_workspace_bytes_hw", "tiny_hotwords", "fp32"): (2046976, 2046464),
    ("fa_paraformer_decoder_workspace_bytes_hw", "tiny_hotwords", "fp16"): (4256768, 2362880),
    ("fa_paraformer_decoder_workspace_bytes_hw", "tiny_hotwords", "fp16x3"): (4951040, 3133952),
    ("fa_paraformer_decoder_workspace_bytes_hw", "tiny_hotwords", "fp16x6"): (5405696, 3468800),
    ("fa_paraformer_decoder_workspace_bytes_hw", "config2", "fp32"): (607781120, 574226432),
    ("fa_paraformer_decoder_workspace_bytes_hw", "config2", "fp16"): (1137575168, 567410688),
    ("fa_paraformer_decoder_workspace_bytes_hw", "config2", "fp16x3"): (1268647168, 725221376),
    ("fa_paraformer_decoder_workspace_bytes_hw", "config2", "fp16x6"): (1399719168, 808321024),
    ("fa_paraformer_decoder_workspace_bytes_hw", "config2_hotwords", "fp32"): (607916544, 607916032),
    ("fa_paraformer_decoder_workspace_bytes_hw", "config2_hotwords", "fp16"): (1154488832, 659919872),
    ("fa_paraformer_decoder_workspace_bytes_hw", "config2_hotwords", "fp16x3"): (1302338048, 842995712),
    ("fa_paraformer_decoder_workspace_bytes_hw", "config2_hotwords", "fp16x6"): (1450187264, 942872576),
    ("fa_sanm_decoder_stack_workspace_bytes", "tiny", "fp32"): (725248, 614400),
    ("fa_sanm_decoder_stack_workspace_bytes", "tiny", "fp16"): (1987840, 989184),
    ("fa_sanm_decoder_stack_workspace_bytes", "tiny", "fp16x3"): (2227456, 1419264),
    ("fa_sanm_decoder_stack_workspace_bytes", "tiny", "fp16x6"): (2227456, 1609728),
    ("fa_sanm_decoder_stack_workspace_bytes", "config2", "fp32"): (209977600, 176422912),
    ("fa_sanm_decoder_stack_workspace_bytes", "config2", "fp16"): (430507264, 227016704),
    ("fa_sanm_decoder_stack_workspace_bytes", "config2", "fp16x3"): (464061696, 294387712),
    ("fa_sanm_decoder_stack_workspace_bytes", "config2", "fp16x6"): (497616128, 347013120),
    ("fa_linear_argmax_workspace_bytes", "tiny", "fp32"): (963328, 962928),
    ("fa_linear_argmax_workspace_bytes", "tiny", "fp16"): (992000, 990720),
    ("fa_linear_argmax_workspace_bytes", "tiny", "fp16x3"): (1019648, 1018368),
    ("fa_linear_argmax_workspace_bytes", "tiny", "fp16x6"): (1047296, 1046016),
    ("fa_linear_argmax_workspace_bytes", "config2", "fp32"): (292159744, 292159488),
    ("fa_linear_argmax_workspace_bytes", "config2", "fp16"): (300549376, 300548096),
    ("fa_linear_argmax_workspace_bytes", "config2", "fp16x3"): (308937984, 308936704),
    ("fa_linear_argmax_workspace_bytes", "config2", "fp16x6"): (317326592, 317325312),
    ("fa_linear_argmax_workspace_bytes", "punc", "fp32"): (414720, 414400),
    ("fa_linear_argmax_workspace_bytes", "punc", "fp16"): (620544, 619264),
    ("fa_linear_argmax_workspace_bytes", "punc", "fp16x3"): (825344, 824064),
    ("fa_linear_argmax_workspace_bytes", "punc", "fp16x6"): (1030144, 1028864),
    ("fa_ctc_greedy_workspace_bytes", "tiny", "fp32"): (11125760, 11125436),
    ("fa_ctc_greedy_workspace_bytes", "tiny", "fp16"): (11240448, 11239168),
    ("fa_ctc_greedy_workspace_bytes", "tiny", "fp16x3"): (11354112, 11352832),
    ("fa_ctc_greedy_workspace_bytes", "tiny", "fp16x6"): (11467776, 11466496),
    ("fa_ctc_greedy_workspace_bytes", "config4", "fp32"): (3232954624, 3232954368),
    ("fa_ctc_greedy_workspace_bytes", "config4", "fp16"): (3265985792, 3265984512),
    ("fa_ctc_greedy_workspace_bytes", "config4", "fp16x3"): (3299015936, 3299014656),
    ("fa_ctc_greedy_workspace_bytes", "config4", "fp16x6"): (3332046080, 3332044800),
    ("fa_attention_tc_workspace_bytes", "tiny", "fp32"): (0, 0),
    ("fa_attention_tc_workspace_bytes", "tiny", "fp16"): (337920, 337920),
    ("fa_attention_tc_workspace_bytes", "tiny", "fp16x3"): (675840, 675840),
    ("fa_attention_tc_workspace_bytes", "tiny", "fp16x6"): (675840, 675840),
    ("fa_attention_tc_workspace_bytes", "config2", "fp32"): (0, 0),
    ("fa_attention_tc_workspace_bytes", "config2", "fp16"): (99090432, 99090432),
    ("fa_attention_tc_workspace_bytes", "config2", "fp16x3"): (198180864, 198180864),
    ("fa_attention_tc_workspace_bytes", "config2", "fp16x6"): (198180864, 198180864),
    ("fa_campplus_workspace_bytes", "tiny", "fp32"): (5130752, 5130496),
    ("fa_campplus_workspace_bytes", "tiny", "fp16"): (5082112, 5080832),
    ("fa_campplus_workspace_bytes", "tiny", "fp16x3"): (5335552, 5334272),
    ("fa_campplus_workspace_bytes", "tiny", "fp16x6"): (5588992, 5587712),
    ("fa_campplus_workspace_bytes", "spk", "fp32"): (166061312, 166061056),
    ("fa_campplus_workspace_bytes", "spk", "fp16"): (164295424, 164294144),
    ("fa_campplus_workspace_bytes", "spk", "fp16x3"): (172358912, 172357632),
    ("fa_campplus_workspace_bytes", "spk", "fp16x6"): (180422400, 180421120),
    ("fa_fsmn_vad_workspace_bytes", "vad_30s", None): (15744512, 15744064),
    ("fa_fsmn_vad_workspace_bytes", "vad_130s", None): (68224512, 68224064),
    ("fa_blstm_tc_scratch_bytes", "tiny", None): (524544, 524544),
    ("fa_blstm_tc_scratch_bytes", "aligner", None): (524544, 524544),
    ("fa_blstm_tc_scratch_bytes", "max", None): (2097408, 2097408),
    # "before": the buffers the handle held for the head (test_timestamp_head_before_is_the_handles_buffers)
    ("fa_timestamp_head_workspace_bytes", "tiny", "fp32"): (8026380, 8026380),
    ("fa_timestamp_head_workspace_bytes", "tiny", "fp16"): (8367372, 8367372),
    ("fa_timestamp_head_workspace_bytes", "tiny", "fp16x3"): (8708364, 8708364),
    ("fa_timestamp_head_workspace_bytes", "tiny", "fp16x6"): (9049356, 9049356),
    ("fa_timestamp_head_workspace_bytes", "config2", "fp32"): (2163212800, 2163212800),
    ("fa_timestamp_head_workspace_bytes", "config2", "fp16"): (2261516800, 2261516800),
    ("fa_timestamp_head_workspace_bytes", "config2", "fp16x3"): (2359820800, 2359820800),
    ("fa_timestamp_head_workspace_bytes", "config2", "fp16x6"): (2458124800, 2458124800),
    ("fa_timestamp_head_workspace_bytes", "aligner", "fp32"): (101900576, 101900576),
    ("fa_timestamp_head_workspace_bytes", "aligner", "fp16"): (106508576, 106508576),
    ("fa_timestamp_head_workspace_bytes", "aligner", "fp16x3"): (111116576, 111116576),
    ("fa_timestamp_head_workspace_bytes", "aligner", "fp16x6"): (115724576, 115724576),
}



def _query(lib, name, args, mode):
    f = getattr(lib, name)
    out = []
    for a in args:
        if a == "m":
            out.append(MODES[mode])
        elif a == "vad":
            out.append(C.byref(_vad()))
        elif a == "cam":
            out.append(C.byref(_cam()))
        else:
            out.append(a)
    return int(f(*out))


def _params():
    for name, shape, args in CASES:
        for mode in (MODES if "m" in args else [None]):
            yield pytest.param(name, shape, args, mode, id="%s-%s-%s" % (name[3:].replace("_workspace_bytes", ""), shape, mode))


@pytest.mark.parametrize("name,shape,args,mode", list(_params()))
def test_workspace_query_value(name, shape, args, mode):
    before, now = VALUES[(name, shape, mode)]
    got = _query(_abi.load(), name, args, mode)
    assert got == now
    assert got <= before
    if mode == "fp32" and name in ("fa_sanm_encoder_workspace_bytes", "fa_cif_predictor_workspace_bytes", "fa_ctc_greedy_workspace_bytes",
                                   "fa_linear_argmax_workspace_bytes"):
        assert before - got < 512              # the fp32 path keeps every buffer: only the headroom and alignment padding went
    if name == "fa_fsmn_vad_workspace_bytes":
        assert before - got < 512 + 192        # ... and VAD's 256-byte slot for 64 bytes of metadata


def test_fp32_decoder_drops_only_the_contextual_slice():
    """Without hotwords the fp32 decoder no longer carves the [x_src_attn ; cx] rows of the contextual bias decoder."""
    for shape, (B, N) in {"tiny": (3, 9), "config2": (64, 128)}.items():
        before, now = VALUES[("fa_paraformer_decoder_workspace_bytes_hw", shape, "fp32")]
        assert 0 <= before - now - B * N * 1024 * 4 < 512


def test_encoder_and_predictor_at_config2():
    """Bench config 2 in fp16x3: the encoder's query (the engine's largest for Paraformer) and the predictor's."""
    assert VALUES[("fa_sanm_encoder_workspace_bytes", "config2", "fp16x3")] == (1855014144, 992804864)
    assert VALUES[("fa_cif_predictor_workspace_bytes", "config2", "fp16x3")] == (458881280, 131728384)
    lib = _abi.load()
    assert lib.fa_sanm_encoder_workspace_bytes(64, 500, _abi.GEMM_F16X3) == 992804864
    assert lib.fa_cif_predictor_workspace_bytes(64, 500, _abi.GEMM_F16X3) == 131728384


@pytest.mark.parametrize("mode", list(MODES))
def test_timestamp_head_before_is_the_handles_buffers(mode):
    """The pinned "before" of the head's query is what the handle reserved for the head when it sequenced the launches itself:
    the payloads of the upsampled rows, the input projections, the BLSTM output, lens x 3 and the recurrence's scratch for at most
    256 sequences, plus the workspace of the larger GEMM (B * 3T rows, K = D)."""
    lib = _abi.load()
    for shape, (B, T, D) in {"tiny": (3, 37, 512), "config2": (64, 500, 512), "aligner": (8, 300, 320)}.items():
        rows = B * 3 * T
        held = rows * (1 + 8 + 2) * D * 4 + B * 4 + lib.fa_blstm_tc_scratch_bytes(min(B, 256)) + \
            lib.fa_linear_workspace_bytes(rows, D, MODES[mode])
        assert VALUES[("fa_timestamp_head_workspace_bytes", shape, mode)][0] == held
    assert lib.fa_timestamp_head_workspace_bytes(0, 37, 512, 3, MODES[mode]) == 0


@pytest.mark.parametrize("mode", list(MODES))
def test_linear_workspace_is_the_operand_split(mode):
    """fa_linear's query: the fp16 planes of x (1 / 2 / 3 for fp16 / x3 / x6) at in_f rounded up to 64, nothing in fp32."""
    lib = _abi.load()
    npl = {"fp32": 0, "fp16": 1, "fp16x3": 2, "fp16x6": 3}[mode]
    for rows, in_f in ((1, 8), (37 * 3, 560), (64 * 500 * 3, 512), (8 * 300 * 3, 320), (200, 1024)):
        assert lib.fa_linear_workspace_bytes(rows, in_f, MODES[mode]) == npl * rows * ((in_f + 63) // 64 * 64) * 2
    assert lib.fa_linear_workspace_bytes(-1, 512, MODES[mode]) == 0
