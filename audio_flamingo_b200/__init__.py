"""audio_flamingo_b200 -- H100-native (sm_90a) implementation of Audio Flamingo 3's audio->text forward path.

Public surface (mirrors the reference's module roles, SURVEY.md 8-b):
    AudioFlamingo3ForConditionalGeneration, AudioFlamingo3Encoder, AudioFlamingo3MultiModalProjector, Qwen2ForCausalLM
    AF3FeatureExtractor (GPU log-mel with the WhisperFeatureExtractor call surface) and the processor's window arithmetic
All compute goes through libaf3b200.so (C ABI in include/af3b200.h); importing this package does not need a GPU,
running it does -- there is no CPU fallback.
"""
from ._lib import AF3Error, lib_path, load as load_library  # noqa: F401


def __getattr__(name):  # lazy: keep `import audio_flamingo_b200` light (torch/transformers only on first use)
    if name in ("AudioFlamingo3ForConditionalGeneration", "MusicFlamingoForConditionalGeneration", "AudioFlamingo3Encoder", "AudioFlamingo3MultiModalProjector",
                "Qwen2ForCausalLM", "AF3KVCache"):
        from . import modeling

        return getattr(modeling, name)
    if name in ("AF3FeatureExtractor", "split_windows", "tokens_per_sample", "expand_audio_tokens", "expand_audio_spans", "left_pad",
                "audio_token_length"):
        from . import processing

        return getattr(processing, name)
    if name == "GatedCrossAttentionLayer":
        from . import xattn

        return xattn.GatedCrossAttentionLayer
    if name in ("shard_rows", "gather_tokens", "plan_kv_capacity", "kv_bytes_per_token"):
        from . import sharding

        return getattr(sharding, name)
    raise AttributeError(name)
