"""kvpress_b200 — the score -> top-k -> gather hot path of NVIDIA/kvpress as hand-written sm_90a
CUDA behind the reference's own press API (BasePress / ScorerPress hooks and the
"kv-press-text-generation" pipeline). See DESIGN.md for scope and INTEGRATION.md for the C ABI.
"""
from kvpress_b200.attention_patch import patch_attention_functions
from kvpress_b200.pipeline import KVPressTextGenerationPipeline
from kvpress_b200.presses.adakv_press import AdaKVPress
from kvpress_b200.presses.base_press import SUPPORTED_MODELS, BasePress
from kvpress_b200.presses.block_press import BlockPress
from kvpress_b200.presses.cam_press import CAMPress
from kvpress_b200.presses.chunk_press import ChunkPress
from kvpress_b200.presses.chunkkv_press import ChunkKVPress
from kvpress_b200.presses.composed_press import ComposedPress
from kvpress_b200.presses.compression_ratio_decoding_press import CompressionRatioDecodingPress
from kvpress_b200.presses.criticalkv_press import CriticalAdaKVPress, CriticalKVPress
from kvpress_b200.presses.cur_press import CURPress
from kvpress_b200.presses.decoding_press import DecodingPress
from kvpress_b200.presses.dms_press import DMSPress
from kvpress_b200.presses.expected_attention_press import ExpectedAttentionPress
from kvpress_b200.presses.expected_attention_with_stats import ExpectedAttentionStatsPress
from kvpress_b200.presses.key_rerotation_press import KeyRerotationPress
from kvpress_b200.presses.keydiff_press import KeyDiffPress
from kvpress_b200.presses.knorm_press import KnormPress
from kvpress_b200.presses.kvzap_press import KVzapConfig, KVzapModel, KVzapPress
from kvpress_b200.presses.lagkv_press import LagKVPress
from kvpress_b200.presses.merging_press import MergingPress
from kvpress_b200.presses.non_causal_attention_press import NonCausalAttnPress
from kvpress_b200.presses.observed_attention_press import ObservedAttentionPress
from kvpress_b200.presses.per_layer_compression_press import PerLayerCompressionPress
from kvpress_b200.presses.prefill_decoding_press import PrefillDecodingPress
from kvpress_b200.presses.pyramidkv_press import PyramidKVPress
from kvpress_b200.presses.random_press import RandomPress
from kvpress_b200.presses.scorer_press import ScorerPress
from kvpress_b200.presses.snapkv_press import SnapKVPress
from kvpress_b200.presses.streaming_llm_press import StreamingLLMPress
from kvpress_b200.presses.finch_press import FinchPress
from kvpress_b200.presses.think_press import ThinKPress
from kvpress_b200.presses.tova_press import TOVAPress

# Like the reference (kvpress/__init__.py:8,52): every attention function of transformers is wrapped at import,
# so head-wise masking (AdaKV) and the cu_seq_lens_k repair after any press shortened a cache are always live.
patch_attention_functions()

__all__ = [
    "BasePress",
    "ScorerPress",
    "KnormPress",
    "SnapKVPress",
    "ExpectedAttentionPress",
    "ExpectedAttentionStatsPress",
    "StreamingLLMPress",
    "TOVAPress",
    "DecodingPress",
    "CAMPress",
    "KVzapPress",
    "KVzapModel",
    "KVzapConfig",
    "DMSPress",
    "KeyRerotationPress",
    "KeyDiffPress",
    "AdaKVPress",
    "CriticalKVPress",
    "CriticalAdaKVPress",
    "ObservedAttentionPress",
    "NonCausalAttnPress",
    "LagKVPress",
    "CURPress",
    "MergingPress",
    "ThinKPress",
    "FinchPress",
    "BlockPress",
    "ChunkPress",
    "ChunkKVPress",
    "ComposedPress",
    "PerLayerCompressionPress",
    "PrefillDecodingPress",
    "CompressionRatioDecodingPress",
    "PyramidKVPress",
    "RandomPress",
    "KVPressTextGenerationPipeline",
    "SUPPORTED_MODELS",
]
