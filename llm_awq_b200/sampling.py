"""tinychat's per-token choice of the next token (tinychat/stream_generators/stream_gen.py: prepare_logits_processor
and the argmax / multinomial that follows it) as one launch of `awq_inference_engine.sample_next_token`.

Only tinychat's gating is restated here: which processors it would build from its generation parameters, and when
it takes the argmax.  The arithmetic is the kernel's (include/b200awq.h, b200awq_sample_next_token)."""
import torch

from .engine import engine


def sample_next_token(logits, output_ids, temp, repeat_penalty, top_p, top_k, n_vocab, generator=None):
    """The next token of each row of `logits` (fp32 [batch, vocab], e.g. the model's `logits[:, -1, :]`), as an int64
    [batch] device tensor.

    temp, repeat_penalty, top_p, top_k and n_vocab are tinychat's generation parameters (`gen_params`); `output_ids`
    are the ids so far (int64 [batch, n] on the logits' device, or None), read only when repeat_penalty > 1.  The
    uniforms of the draw come from `generator` (a torch.Generator on the logits' device; None: the default one)."""
    greedy = temp < 1e-5 or top_p < 1e-8
    if top_k <= 0:
        top_k = n_vocab
    temperature = temp if temp >= 1e-5 and temp != 1.0 else 1.0
    penalty = repeat_penalty if repeat_penalty > 1.0 else 1.0
    top_p = top_p if 1e-8 <= top_p < 1.0 else 1.0
    prev = output_ids if penalty > 1.0 else None
    uniforms = None
    if not greedy:
        uniforms = torch.rand(logits.shape[0], generator=generator, device=logits.device, dtype=torch.float32)
    return engine().sample_next_token(logits, prev, temperature, penalty, top_p, min(top_k, 2 ** 31 - 1), greedy,
                                      uniforms)
