"""The "kv-press-text-generation" pipeline.

API-stable mirror of `kvpress/pipeline.py:25-331`: same task name, same call
keywords (`question`, `questions`, `answer_prefix`, `press`, `max_new_tokens`, `max_context_length`,
`enable_thinking`, `cache`), same result keys (`answer` / `answers`), same two debug log lines.
Flow: tokenise context and questions separately, prefill the context once under `press(model)` so
the press compacts every layer's cache, then answer each question greedily on top of the compacted
cache and strip the answer tokens from the cache afterwards.
"""
from __future__ import annotations

import contextlib
import logging
from typing import Optional

import torch
from transformers import AutoModelForCausalLM, Cache, DynamicCache, Pipeline
from transformers.pipelines import PIPELINE_REGISTRY

from kvpress_b200.presses.base_press import BasePress
from kvpress_b200.presses.decoding_press import DecodingPress
from kvpress_b200.presses.dms_press import DMSPress
from kvpress_b200.presses.finch_press import FinchPress
from kvpress_b200.presses.key_rerotation_press import KeyRerotationPress
from kvpress_b200.presses.prefill_decoding_press import PrefillDecodingPress

logger = logging.getLogger(__name__)


class KVPressTextGenerationPipeline(Pipeline):
    """`pipeline("kv-press-text-generation", model=...)(context, question=..., press=...)`"""

    def _sanitize_parameters(
        self,
        question: Optional[str] = None,
        questions: Optional[list[str]] = None,
        answer_prefix: Optional[str] = None,
        press: Optional[BasePress] = None,
        max_new_tokens: int = 50,
        max_context_length: Optional[int] = None,
        enable_thinking: bool = False,
        cache: Optional[Cache] = None,
        **kwargs,
    ):
        assert question is None or questions is None, "Either question or questions should be provided, not both."
        single = questions is None
        if questions is None:
            questions = [question] if question else [""]
        if max_context_length is None:
            max_context_length = min(self.tokenizer.model_max_length, int(1e10))
        preprocess_kwargs = {
            "questions": questions,
            "answer_prefix": answer_prefix or "",
            "max_context_length": max_context_length,
            "enable_thinking": enable_thinking,
        }
        forward_kwargs = {"press": press, "max_new_tokens": max_new_tokens, "cache": cache}
        return preprocess_kwargs, forward_kwargs, {"single_question": single}

    def preprocess(self, context: str, questions: list[str], answer_prefix: str, max_context_length: int,
                   enable_thinking: bool = False):
        """Split the chat-templated prompt into a context part and a per-question suffix, tokenise both."""
        tok = self.tokenizer
        if tok.chat_template is None:
            context = (getattr(tok, "bos_token", "") or "") + context
            question_suffix = "\n"
        else:
            marker = "#" * (len(context) + 10)  # cannot occur in the context
            templated = tok.apply_chat_template(
                [{"role": "user", "content": context + marker}],
                add_generation_prompt=True,
                tokenize=False,
                enable_thinking=enable_thinking,
            )
            context, question_suffix = templated.split(marker)
        context_ids = tok.encode(context, return_tensors="pt", add_special_tokens=False)
        question_ids = [
            tok.encode(q + question_suffix + answer_prefix, return_tensors="pt", add_special_tokens=False)
            for q in questions
        ]
        if context_ids.shape[1] > max_context_length:
            logger.warning(
                f"Context length has been truncated from {context_ids.shape[1]} to {max_context_length} tokens.")
            context_ids = context_ids[:, :max_context_length]
        return {"context_ids": context_ids, "questions_ids": question_ids}

    def _forward(self, input_tensors, max_new_tokens: int = 50, press: Optional[BasePress] = None,
                 cache: Optional[Cache] = None):
        # pipeline.py:202-233 of the reference: a DecodingPress is live only while generating, a
        # PrefillDecodingPress and a DMSPress with decoding=True in both phases, everything else only during prefill.
        # Unlike the reference, a decoding DMSPress also refuses several questions: the positions it masks while
        # answering one would outlive _remove_answer_from_cache and mask the next question's tokens.
        decoding = isinstance(press, (DecodingPress, PrefillDecodingPress)) or (
            isinstance(press, DMSPress) and press.decoding)
        prefilling = press is not None and not isinstance(press, DecodingPress)
        if decoding and len(input_tensors["questions_ids"]) > 1:
            raise ValueError("DecodingPress is not compatible with multiple questions. Please specify a single question.")

        context_ids = input_tensors["context_ids"].to(self.model.device)
        context_length = context_ids.shape[1]
        if cache is None:
            cache = DynamicCache()

        prefill_ctx = press(self.model) if prefilling else contextlib.nullcontext()
        with prefill_ctx:
            self.model.model(input_ids=context_ids, past_key_values=cache)  # no lm_head during prefill
            logger.debug(f"Context Length: {context_length}")
            logger.debug(f"Compressed Context Length: {cache.get_seq_length()}")

        decode_ctx = press(self.model) if decoding else contextlib.nullcontext()
        answers = []
        with decode_ctx:
            for question_ids in input_tensors["questions_ids"]:
                if isinstance(press, KeyRerotationPress) or (isinstance(press, FinchPress) and press.rerotate_keys):
                    # pipeline.py:231-237 of the reference: the kept keys were re-rotated to positions
                    # 0..n_kept-1, so question and answer continue from the COMPRESSED length
                    context_length = cache.get_seq_length()
                lengths_before = [cache.get_seq_length(i) for i in range(len(cache))]
                answers.append(
                    self.generate_answer(
                        question_ids=question_ids.to(self.model.device),
                        cache=cache,
                        context_length=context_length,
                        max_new_tokens=max_new_tokens,
                    )
                )
                self._remove_answer_from_cache(cache, lengths_before)
        return answers

    def _remove_answer_from_cache(self, cache: Cache, cache_seq_lengths: list[int]):
        for layer_idx, length in enumerate(cache_seq_lengths):
            layer = cache.layers[layer_idx]
            layer.keys = layer.keys[:, :, :length]
            layer.values = layer.values[:, :, :length]

    def generate_answer(self, question_ids: torch.Tensor, cache: Cache, context_length: int, max_new_tokens: int) -> str:
        """Greedy decoding of one answer; positions continue from the ORIGINAL context length."""
        device = self.model.device
        position_ids = torch.arange(context_length, context_length + question_ids.shape[1], device=device).unsqueeze(0)
        outputs = self.model(input_ids=question_ids.to(device), past_key_values=cache, position_ids=position_ids,
                             logits_to_keep=1)
        next_position = position_ids[:, -1:] + 1
        generated = [outputs.logits[0, -1].argmax()]

        stop_ids = self.model.generation_config.eos_token_id
        if not isinstance(stop_ids, list):
            stop_ids = [stop_ids]
        for step in range(max_new_tokens - 1):
            outputs = self.model(input_ids=generated[-1].view(1, 1), past_key_values=cache,
                                 position_ids=next_position + step)
            token = outputs.logits[0, -1].argmax()
            generated.append(token)
            if token.item() in stop_ids:
                break
        return str(self.tokenizer.decode(torch.stack(generated), skip_special_tokens=True))

    def postprocess(self, model_outputs, single_question):
        return {"answer": model_outputs[0]} if single_question else {"answers": model_outputs}


PIPELINE_REGISTRY.register_pipeline(
    "kv-press-text-generation",
    pipeline_class=KVPressTextGenerationPipeline,
    pt_model=AutoModelForCausalLM,
)
