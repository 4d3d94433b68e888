"""funasr_b200 — H100-native (sm_90a) backend for FunASR's offline Paraformer hot path.

Importing this package registers the drop-in plugin classes (ParaformerB200, WavFrontendB200, SANMEncoderB200,
CifPredictorV2B200, ParaformerSANMDecoderB200) — into ``funasr.register.tables`` when FunASR is imported, else into
a local table with the same API.  ``funasr_b200.install(override_reference_keys=True)`` additionally re-points the
reference's own keys at these classes so an unmodified FunASR config runs on this backend.
"""
from .registry import get_tables, install, register  # noqa: F401
from .synth import PARAFORMER_LARGE, PARAFORMER_TINY, ParaformerConfig  # noqa: F401
from . import modules  # noqa: F401  (registers the classes)
from .modules import (CifPredictorV2B200, ParaformerB200, ParaformerSANMDecoderB200, SANMEncoderB200,  # noqa: F401
                      SenseVoiceEncoderSmallB200, SenseVoiceSmallB200, WavFrontendB200, load_cmvn,
                      ContextualParaformerB200, ContextualParaformerDecoderB200, BiCifParaformerB200, CifPredictorV3B200,
                      SeacoParaformerB200)
from .engine import FrontendEngine, ParaformerEngine, SenseVoiceEngine  # noqa: F401
from .synth import SENSEVOICE_SMALL, SENSEVOICE_TINY, SenseVoiceConfig  # noqa: F401
from .sharding import shard_utterances, gather_token_ids, ShardedRunner  # noqa: F401
from .batching import bucket_by_length, padding_efficiency, run_bucketed  # noqa: F401
from .vad import VadOptions, detect_segments, detect_segments_native, merge_vad  # noqa: F401
from .vad_model import FSMNB200, FsmnVADStreamingB200, VadEngine, WavFrontendOnlineB200  # noqa: F401
from .long_audio import LongAudioPipeline, merge_results, pack_segments  # noqa: F401
from .punc import CTTransformerB200, PuncEngine, split_to_mini_sentence, split_words  # noqa: F401
from .audio import decode_pcm, load_audio, parse_wav_header  # noqa: F401
from .hotwords import generate_hotwords_list, load_seg_dict, seg_tokenize  # noqa: F401
from .campplus import CAMPPlusB200, CampplusEngine  # noqa: F401
from . import diarization  # noqa: F401

__version__ = "0.1.0"
