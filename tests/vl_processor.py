"""An offline Qwen2.5-VL processor for the System-2 image tests: the real `Qwen2_5_VLProcessor` (text expansion,
Qwen2VLImageProcessorPil, chat template rendering) around a word-level tokenizer whose vocabulary covers every id the
tiny model can generate, so generated ids decode to text and that text tokenises back to the same ids."""
import functools

import pytest

VOCAB = 152064
SPECIAL = {151643: "<|endoftext|>", 151644: "<|im_start|>", 151645: "<|im_end|>", 151652: "<|vision_start|>",
           151653: "<|vision_end|>", 151655: "<|image_pad|>", 151656: "<|video_pad|>"}
CHAT_TEMPLATE = (
    "{% for m in messages %}<|im_start|>{{ m['role'] }}\n"
    "{% for c in m['content'] %}{% if c['type'] == 'image' %}<|vision_start|><|image_pad|><|vision_end|>"
    "{% else %}{{ c['text'] }}{% endif %}{% endfor %}<|im_end|>\n{% endfor %}"
    "{% if add_generation_prompt %}<|im_start|>assistant\n{% endif %}")
_AZ = "abcdefghijklmnopqrstuvwxyz"


def word(i):
    """Token i of the word-level vocabulary: four letters (no digits, so an answer is never read as a pixel goal)."""
    return "".join(_AZ[(i // 26 ** k) % 26] for k in range(3, -1, -1))


def qwen_processor(**image_kwargs):
    """Qwen2_5_VLProcessor with Qwen2VLImageProcessorPil(**image_kwargs); skips the test without transformers 5."""
    pytest.importorskip("tokenizers")
    pytest.importorskip("transformers.models.qwen2_vl.image_processing_pil_qwen2_vl")
    return _processor(tuple(sorted(image_kwargs.items())))


@functools.lru_cache(maxsize=None)
def _processor(image_kwargs):
    import transformers.models.qwen2_vl.image_processing_pil_qwen2_vl as ipm
    from tokenizers import Tokenizer, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast, Qwen2_5_VLProcessor, Qwen2VLVideoProcessor
    vocab = {word(i): i for i in range(VOCAB) if i not in SPECIAL}
    vocab.update({t: i for i, t in SPECIAL.items()})
    tk = Tokenizer(models.WordLevel(vocab, unk_token=word(0)))
    tk.pre_tokenizer = pre_tokenizers.Whitespace()
    tok = PreTrainedTokenizerFast(tokenizer_object=tk, unk_token=word(0), eos_token="<|im_end|>",
                                  pad_token="<|endoftext|>", additional_special_tokens=list(SPECIAL.values()))
    return Qwen2_5_VLProcessor(image_processor=ipm.Qwen2VLImageProcessorPil(**dict(image_kwargs)), tokenizer=tok,
                               video_processor=Qwen2VLVideoProcessor(), chat_template=CHAT_TEMPLATE)
