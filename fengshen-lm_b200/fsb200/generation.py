"""Model-agnostic generation controller: the token-selection loop of transformers' `GenerationMixin.generate` (HF 5.5.0,
generation/utils.py `_sample` and `_beam_search`) on top of a model-provided step function.

A model's `generate` resolves the options with `resolve(...)` (LLaMA: from its own keyword defaults), prepares its caches
for `rows = batch * cfg.expand` sequences, and calls `run(step, seqs, cfg)`. The step contract is

    step(next_tokens, beam_reorder) -> fp32 logits [rows, V] of the last position of every row
      * step(None, None): the prefill (the prompt rows, already expanded);
      * step(tokens [rows], reorder [rows] or None): first gather every cache row from `reorder` (beam search), then append
        `tokens` and return the next logits.
      * the returned logits are a FRESH tensor that the model never writes again: the loop keeps them (`scores`, and greedy
        without a penalty processes them into the very same tensor), so a step that computes into a static buffer (a
        CUDA-graph replay, fsb200/decode_graph.py) returns a clone of it. `tokens` and `reorder` are only read during the
        call; the step copies what it needs.

Everything here is host-side PyTorch on whatever device the logits live on; the model does the GPU work.

Implemented: greedy; sampling with temperature / top_k / top_p (HF's default top_k of 50 applies); repetition_penalty;
num_return_sequences; eos_token_id (int or list) / pad_token_id with finished rows padded; max_length / max_new_tokens; beam
search with num_beams / length_penalty / early_stopping (True, False or "never") / num_return_sequences <= num_beams, its
processors applied to log-probabilities; return_dict_in_generate with sequences, scores (output_scores) and, for beam search,
sequences_scores. Any other generation keyword that would change the result raises NotImplementedError naming it.
"""
from types import SimpleNamespace

import torch

_SUPPORTED = {"max_length", "max_new_tokens", "do_sample", "temperature", "top_k", "top_p", "repetition_penalty",
              "num_beams", "num_return_sequences", "length_penalty", "early_stopping", "eos_token_id", "pad_token_id",
              "decoder_start_token_id", "return_dict_in_generate", "output_scores"}
# keywords accepted at the value that makes them inert (HF's defaults); any other value is refused
_INERT = {"num_beam_groups": 1, "no_repeat_ngram_size": 0, "encoder_no_repeat_ngram_size": 0, "min_length": 0,
          "min_new_tokens": 0, "diversity_penalty": 0.0, "typical_p": 1.0, "output_attentions": False,
          "output_hidden_states": False, "output_logits": False, "use_cache": True, "synced_gpus": False,
          "renormalize_logits": False, "remove_invalid_values": False, "bos_token_id": None}


def resolve(model_config, kwargs, input_len, is_encoder_decoder):
    """Merge `kwargs` over the defaults HF's GenerationConfig derives from the model config. input_len is the length of the
    sequences the loop extends (the prompt for a decoder-only model, 1 — the start token — for an encoder-decoder)."""
    for k, v in kwargs.items():
        if k in _SUPPORTED:
            continue
        if v is None or (k in _INERT and v == _INERT[k]):
            continue
        raise NotImplementedError(f"fsb200 generate: `{k}` is not implemented (got {v!r})")
    g = lambda k, d=None: kwargs[k] if kwargs.get(k) is not None else getattr(model_config, k, d)   # noqa: E731
    c = SimpleNamespace()
    c.do_sample = bool(kwargs.get("do_sample") or False)
    c.temperature = float(kwargs.get("temperature") if kwargs.get("temperature") is not None else 1.0)
    c.top_k = int(kwargs.get("top_k") if kwargs.get("top_k") is not None else 50)
    c.top_p = float(kwargs.get("top_p") if kwargs.get("top_p") is not None else 1.0)
    c.repetition_penalty = float(kwargs.get("repetition_penalty") if kwargs.get("repetition_penalty") is not None else 1.0)
    c.num_beams = int(kwargs.get("num_beams") or 1)
    c.num_return_sequences = int(kwargs.get("num_return_sequences") or 1)
    c.length_penalty = float(kwargs.get("length_penalty") if kwargs.get("length_penalty") is not None else 1.0)
    c.early_stopping = kwargs.get("early_stopping") if kwargs.get("early_stopping") is not None else False
    c.return_dict = bool(kwargs.get("return_dict_in_generate") or False)
    c.output_scores = bool(kwargs.get("output_scores") or False)
    eos = g("eos_token_id")
    c.eos = None if eos is None else ([int(eos)] if isinstance(eos, int) else [int(e) for e in eos])
    pad = g("pad_token_id")
    c.pad = int(pad) if pad is not None else (c.eos[0] if c.eos else None)   # HF: pad defaults to the first eos
    if is_encoder_decoder:
        start = g("decoder_start_token_id")
        c.start = int(start) if start is not None else (c.pad if c.pad is not None else 0)
    if kwargs.get("max_new_tokens") is not None:
        c.max_length = input_len + int(kwargs["max_new_tokens"])
    elif kwargs.get("max_length") is not None:
        c.max_length = int(kwargs["max_length"])
    else:   # HF 5.x: the default max_length of 20 counts NEW tokens, capped at the position table
        c.max_length = 20 + input_len
        npos = getattr(model_config, "max_position_embeddings", None)
        if npos is not None:
            c.max_length = min(c.max_length, int(npos))
    if c.num_beams > 1:
        if c.do_sample:
            raise NotImplementedError("fsb200 generate: beam sampling (`do_sample=True` with `num_beams` > 1) is not implemented")
        if c.num_return_sequences > c.num_beams:
            raise ValueError("fsb200 generate: `num_return_sequences` has to be smaller or equal to `num_beams`")
        c.expand = c.num_beams
    else:
        if not c.do_sample and c.num_return_sequences > 1:
            raise ValueError("fsb200 generate: greedy search with `num_return_sequences` > 1 returns identical rows; "
                             "set do_sample=True or num_beams")
        c.expand = c.num_return_sequences
    return c


def default_attention_mask(ids, pad, eos):
    """HF `_prepare_attention_mask_for_generation`: mask out pad tokens when the pad id occurs and differs from every eos."""
    if pad is not None and bool((ids == pad).any()) and (eos is None or pad not in eos):
        return (ids != pad).long()
    return torch.ones_like(ids)


def process(logits, seqs, do_sample, temperature, top_k, top_p, repetition_penalty, min_keep=1):
    """HF logits-processor order: repetition penalty -> (sampling only) temperature -> top-k -> top-p."""
    if repetition_penalty != 1.0:
        seen = torch.gather(logits, 1, seqs)
        seen = torch.where(seen < 0, seen * repetition_penalty, seen / repetition_penalty)
        logits = logits.scatter(1, seqs, seen)
    if not do_sample:
        return logits
    if temperature != 1.0:
        logits = logits / temperature
    if top_k and top_k > 0:
        kth = torch.topk(logits, min(max(top_k, min_keep), logits.shape[-1]), dim=-1).values[:, -1:]
        logits = logits.masked_fill(logits < kth, float("-inf"))
    if top_p < 1.0:
        srt, idx = torch.sort(logits, descending=False, dim=-1)
        cum = torch.softmax(srt, -1).cumsum(-1)
        remove = cum <= (1.0 - top_p)
        remove[:, -min_keep:] = False
        logits = logits.masked_fill(remove.scatter(1, idx, remove), float("-inf"))
    return logits


def run(step, seqs, c, generator=None):
    """seqs: int64 [rows, L0] (rows = batch * c.expand, already expanded). Returns the sequences [rows', <= max_length], or
    a namespace with .sequences / .scores / .sequences_scores when c.return_dict."""
    if c.num_beams > 1:
        return _beam_search(step, seqs, c)
    return _sample(step, seqs, c, generator)


def _sample(step, seqs, c, generator):
    eos = None if c.eos is None else torch.tensor(c.eos, device=seqs.device)
    unfinished = torch.ones(seqs.shape[0], dtype=torch.bool, device=seqs.device)
    scores = []
    logits = step(None, None)
    while True:
        s = process(logits, seqs, c.do_sample, c.temperature, c.top_k, c.top_p, c.repetition_penalty)
        if c.output_scores:
            scores.append(s)
        if c.do_sample:
            nxt = torch.multinomial(torch.softmax(s, -1), 1, generator=generator).squeeze(1)
        else:
            nxt = s.argmax(-1)
        if eos is not None:
            nxt = torch.where(unfinished, nxt, torch.full_like(nxt, c.pad))
        seqs = torch.cat([seqs, nxt[:, None]], dim=1)
        done = torch.full_like(unfinished, seqs.shape[1] >= c.max_length)
        if eos is not None:
            done = done | torch.isin(nxt, eos)
        unfinished = unfinished & ~done
        if not bool(unfinished.any()):
            break
        logits = step(nxt, None)
    if not c.return_dict:
        return seqs
    return SimpleNamespace(sequences=seqs, scores=tuple(scores) if c.output_scores else None, sequences_scores=None)


def _beam_search(step, seqs, c):
    """HF 5.5.0 `_beam_search` (generation/utils.py:3076-3409 with its helpers :2844-3072), greedy beams."""
    dev = seqs.device
    nb = c.num_beams
    rows, L0 = seqs.shape
    B = rows // nb
    n_eos = len(c.eos) if c.eos is not None else 0
    keep = max(2, 1 + n_eos) * nb
    top_mask = torch.arange(keep, device=dev) < nb
    eos = None if c.eos is None else torch.tensor(c.eos, device=dev)
    fill = (c.pad if c.pad else c.eos[0]) if c.eos is not None else -1   # `pad or eos[0] if eos is not None else -1`
    T = max(c.max_length, L0 + 1)
    run_seq = torch.full((B, nb, T), fill, dtype=torch.int64, device=dev)
    run_seq[:, :, :L0] = seqs.view(B, nb, L0)
    fin_seq = run_seq.clone()
    run_score = torch.zeros((B, nb), dtype=torch.float32, device=dev)
    run_score[:, 1:] = -1e9
    fin_score = torch.full((B, nb), -1e9, dtype=torch.float32, device=dev)
    run_len = torch.zeros((B, nb), dtype=torch.int64, device=dev)   # generated tokens per beam (HF: beam_indices != -1)
    fin_len = run_len.clone()
    fin = torch.zeros((B, nb), dtype=torch.bool, device=dev)
    improvable = torch.ones((B, 1), dtype=torch.bool, device=dev)
    gather = lambda t, i: torch.take_along_dim(t, i.view(i.shape + (1,) * (t.dim() - 2)), dim=1)   # noqa: E731
    all_scores = []
    cur = L0
    flat = seqs
    logits = step(None, None)
    while True:
        V = logits.shape[-1]
        logp = torch.log_softmax(logits.float(), dim=-1)
        logp = process(logp, flat, False, 1.0, 0, 1.0, c.repetition_penalty)
        if c.output_scores:
            all_scores.append(logp.clone())
        acc = (logp.view(B, nb, V) + run_score[:, :, None]).view(B, nb * V)
        # top-K continuations over all beams of a batch item
        tk_lp, tk_idx = torch.topk(acc, k=keep)
        src = tk_idx // V
        tk_seq = gather(run_seq, src)
        tk_seq[:, :, cur] = tk_idx % V
        tk_len = gather(run_len, src) + 1
        hits = torch.full((B, keep), cur + 1 >= c.max_length, dtype=torch.bool, device=dev)
        if eos is not None:
            hits = hits | torch.isin(tk_seq[:, :, cur], eos)
        # running beams for the next step: the best `nb` that did not just finish
        tk_run = tk_lp + hits.float() * -1.0e9
        nxt_i = torch.topk(tk_run, k=nb)[1]
        new_seq, new_score, new_len = gather(tk_seq, nxt_i), gather(tk_run, nxt_i), gather(tk_len, nxt_i)
        reorder = (gather(src, nxt_i) + torch.arange(B, device=dev)[:, None] * nb).view(-1)
        # finished hypotheses: merge the newly finished top-`nb` candidates into the kept ones
        just = hits & top_mask[None, :]
        f_lp = tk_lp / ((cur + 1 - L0) ** c.length_penalty)
        full = torch.all(fin, dim=-1, keepdim=True) & (c.early_stopping is True)
        f_lp = f_lp + full.float() * -1.0e9
        f_lp = f_lp + (~improvable).float() * -1.0e9
        f_lp = f_lp + (~just) * -1.0e9
        m_score = torch.cat((fin_score, f_lp), dim=1)
        top = torch.topk(m_score, k=nb)[1]
        fin_seq = gather(torch.cat((fin_seq, tk_seq), dim=1), top)
        fin_score = gather(m_score, top)
        fin_len = gather(torch.cat((fin_len, tk_len), dim=1), top)
        fin = gather(torch.cat((fin, just), dim=1), top)
        run_seq, run_score, run_len = new_seq, new_score, new_len
        cur += 1
        # can a running beam still beat the worst finished one?
        if c.early_stopping == "never" and c.length_penalty > 0.0:
            best_len = c.max_length - L0
        else:
            best_len = cur - L0
        best_run = run_score[:, :1] / (best_len ** c.length_penalty)
        worst_fin = torch.where(fin, torch.min(fin_score, dim=1, keepdim=True)[0], -1.0e9)
        improvable = improvable & torch.any(best_run > worst_fin, dim=-1, keepdim=True)
        go = bool(improvable.any()) and not (bool(fin.all()) and c.early_stopping is True) and not bool(hits.all()) \
            and cur < T
        if not go:
            break
        flat = run_seq[:, :, :cur].reshape(B * nb, cur)
        logits = step(flat[:, -1].contiguous(), reorder)
    nrs = c.num_return_sequences
    out = fin_seq[:, :nrs].reshape(B * nrs, T)
    out = out[:, :L0 + int(fin_len[:, :nrs].max())]
    if not c.return_dict:
        return out
    return SimpleNamespace(sequences=out, scores=tuple(all_scores) if c.output_scores else None,
                           sequences_scores=fin_score[:, :nrs].reshape(-1) if c.output_scores else None)
