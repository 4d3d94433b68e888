"""Plugin registry surface.

When FunASR itself is importable, classes register straight into ``funasr.register.tables`` (the reference's
RegisterTables singleton, funasr/register.py:92) so ``AutoModel(model="ParaformerB200", ...)`` finds them.
Without FunASR (e.g. the GPU box of this project) a local object with the same ``register`` decorator API and the
same table names (funasr/register.py:11-24, :49-89) is used, so the classes and tests behave identically.
"""
from __future__ import annotations

import sys

TABLE_NAMES = (
    "model_classes", "frontend_classes", "specaug_classes", "normalize_classes", "encoder_classes",
    "decoder_classes", "joint_network_classes", "predictor_classes", "stride_conv_classes", "tokenizer_classes",
    "dataloader_classes", "batch_sampler_classes", "dataset_classes", "index_ds_classes",
)


class LocalRegisterTables:
    """Same behaviour as funasr.register.RegisterTables.register: last writer wins (register.py:65-70)."""

    def __init__(self):
        for n in TABLE_NAMES:
            setattr(self, n, {})

    def register(self, register_tables_key: str, key=None):
        def decorator(target_class):
            if not hasattr(self, register_tables_key):
                setattr(self, register_tables_key, {})
            table = getattr(self, register_tables_key)
            table[key if key is not None else target_class.__name__] = target_class
            return target_class
        return decorator


_local = LocalRegisterTables()


def get_tables():
    """The reference's tables if `funasr.register` is already imported / importable cheaply, else the local ones."""
    mod = sys.modules.get("funasr.register")
    if mod is not None and hasattr(mod, "tables"):
        return mod.tables
    return _local


def register(table: str, key: str):
    """Decorator registering into the local tables now and into funasr's tables when present (see install())."""
    def decorator(cls):
        _local.register(table, key)(cls)
        _PENDING.append((table, key, cls))
        t = get_tables()
        if t is not _local:
            t.register(table, key)(cls)
        return cls
    return decorator


_PENDING = []

# reference key -> our key, for override_reference_keys()
DROP_IN_KEYS = {
    ("model_classes", "Paraformer"): "ParaformerB200",
    ("frontend_classes", "WavFrontend"): "WavFrontendB200",
    ("frontend_classes", "wav_frontend"): "WavFrontendB200",
    ("encoder_classes", "SANMEncoder"): "SANMEncoderB200",
    ("predictor_classes", "CifPredictorV2"): "CifPredictorV2B200",
    ("predictor_classes", "CifPredictorV3"): "CifPredictorV3B200",
    ("model_classes", "BiCifParaformer"): "BiCifParaformerB200",
    ("model_classes", "SeacoParaformer"): "SeacoParaformerB200",
    ("model_classes", "FsmnVADStreaming"): "FsmnVADStreamingB200",
    ("model_classes", "CTTransformer"): "CTTransformerB200",
    ("encoder_classes", "FSMN"): "FSMNB200",
    ("frontend_classes", "WavFrontendOnline"): "WavFrontendOnlineB200",
    ("model_classes", "ContextualParaformer"): "ContextualParaformerB200",
    ("decoder_classes", "ContextualParaformerDecoder"): "ContextualParaformerDecoderB200",
    ("model_classes", "SenseVoiceSmall"): "SenseVoiceSmallB200",
    ("encoder_classes", "SenseVoiceEncoderSmall"): "SenseVoiceEncoderSmallB200",
    ("decoder_classes", "ParaformerSANMDecoder"): "ParaformerSANMDecoderB200",
    ("model_classes", "CAMPPlus"): "CAMPPlusB200",
    ("model_classes", "MonotonicAligner"): "MonotonicAlignerB200",
}


def install(override_reference_keys: bool = False):
    """(Re-)register every funasr_b200 class into funasr.register.tables (call after `import funasr`).

    With override_reference_keys=True the reference's own keys ("Paraformer", "WavFrontend", "SANMEncoder",
    "CifPredictorV2", "ParaformerSANMDecoder") are re-pointed at this backend's classes — registration is
    last-writer-wins (funasr/register.py:65-70) — so an unmodified config selects this backend.
    """
    t = get_tables()
    for table, key, cls in _PENDING:
        t.register(table, key)(cls)
    if override_reference_keys:
        for (table, ref_key), ours in DROP_IN_KEYS.items():
            t.register(table, ref_key)(getattr(_local, table)[ours])
    return t
