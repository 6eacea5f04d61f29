"""Request/response shim for the vLLM surface of the reference (demo/demo_vllm.py:18-63,
chatts/utils/llm_utils.py:147-190): ``LLM(model=...).generate([{"prompt": str, "multi_modal_data":
{"timeseries": [...]}}], SamplingParams(...)) -> outputs[i].outputs[0].text``.

The reference's plugin file targets vllm 0.8.5 internals that no longer exist (SURVEY.md §8b); this shim
keeps the REQUEST SHAPE and drives the native engine directly instead of vLLM's plugin ABI."""
from dataclasses import dataclass, field

import numpy as np
import torch

from . import logit_proc as lpmodp
from . import logprobs as lpmod
from .config import ChatTSConfig
from .model import ChatTSForCausalLM
from .processor import ChatTSProcessor, SimpleTokenizer
from .structured import StructuredOutputsParams, resolve as _resolve_structured  # noqa: F401  (StructuredOutputsParams is public here)

MAX_TS_PER_PROMPT = 50      # chatts_vllm.py:219-220


@dataclass
class SamplingParams:
    """The fields the reference's callers set (llm_utils.py:153: temperature, top_p, max_tokens, stop_token_ids, stop, n;
    demo/demo_vllm.py:24)."""
    max_tokens: int = 16
    temperature: float = 0.0
    top_p: float = 1.0
    top_k: int = 0
    stop_token_ids: list = field(default_factory=list)
    stop: list = field(default_factory=list)          # stop STRINGS: the text is cut before the first occurrence
    n: int = 1                                        # completions per request (temperature > 0: independent seeds)
    ignore_eos: bool = False
    seed: int = None
    repetition_penalty: float = 1.0                   # vLLM SamplingParams.repetition_penalty (prompt + generated tokens)
    logprobs: int = None                              # 0..20: logprob of every generated token plus its top-k (single GPU)
    prompt_logprobs: int = None                       # 0..20: the same for every prompt token after the first (single GPU)
    structured_outputs: StructuredOutputsParams = None  # choice / regex constraint on the output (a dict of its fields is accepted)
    presence_penalty: float = 0.0                     # [-2, 2]: subtracted once from every token the output already holds
    frequency_penalty: float = 0.0                    # [-2, 2]: subtracted per occurrence in the output
    logit_bias: dict = None                           # {token id (int or str): bias}, clamped to [-100, 100]
    allowed_token_ids: list = None                    # only these ids may be generated
    min_tokens: int = 0                               # stop ids and stop strings do not end the output before this many tokens

    def __post_init__(self):
        procs = lpmodp.resolve(self.presence_penalty, self.frequency_penalty, self.repetition_penalty, self.logit_bias,
                               self.allowed_token_ids, self.min_tokens, self.max_tokens)
        if procs is not None:
            self.logit_bias = procs.logit_bias
        lpmod.check_k(self.logprobs, "logprobs")
        lpmod.check_k(self.prompt_logprobs, "prompt_logprobs")
        self.structured_outputs = _resolve_structured(self.structured_outputs)
        if self.structured_outputs is not None and self.ignore_eos:
            raise ValueError("structured_outputs end the output with a stop id: they cannot be combined with ignore_eos")


@dataclass
class Logprob:
    """vLLM's Logprob: the log probability of a token, its rank (1 + the number of tokens with a larger logit), its text."""
    logprob: float
    rank: int = None
    decoded_token: str = None


@dataclass
class CompletionOutput:
    text: str
    token_ids: list
    finish_reason: str = None     # "stop" (EOS / stop id / stop string) or "length"
    logprobs: list = None         # SamplingParams.logprobs: per kept token, {id: Logprob} of the token and its top-k
    cumulative_logprob: float = None


def logprob_dict(token, logprob, rank, top_ids, top_lps, tokenizer):
    """{id: Logprob} of a token and its top-k (k or k + 1 entries).  A top-k entry's rank is 1 + the number of entries with a larger
    logprob, all of which are in the top-k."""
    d = {int(token): Logprob(float(logprob), int(rank), decode_text(tokenizer, [int(token)]))}
    for i, lp in zip(top_ids, top_lps):
        if int(i) >= 0 and int(i) not in d:
            d[int(i)] = Logprob(float(lp), 1 + sum(1 for x in top_lps if x > lp), decode_text(tokenizer, [int(i)]))
    return d


def completion_logprobs(res, row, n_tokens, tokens, tokenizer):
    """(logprobs, cumulative_logprob) of the first n_tokens generated tokens of ``row`` of a GenerationLogprobs."""
    out = [logprob_dict(tokens[j], res.logprobs[row, j], res.ranks[row, j], res.top_ids[row, j], res.top_logprobs[row, j], tokenizer)
           for j in range(n_tokens)]
    return out, float(sum(float(res.logprobs[row, j]) for j in range(n_tokens)))


def prompt_logprob_dicts(entries, tokenizer):
    """RequestOutput.prompt_logprobs from GenerationLogprobs.prompt[row]: None, or {id: Logprob} of the token and its top-k."""
    return [None if e is None else logprob_dict(e.token_id, e.logprob, e.rank, e.top_ids, e.top_logprobs, tokenizer) for e in entries]


def tokens_before_stop_string(tokenizer, tokens, stops, min_tokens=0):
    """The number of leading tokens whose text first contains a stop string (all of them when none does): the tokens the cut text
    came from, the one that completed the stop string included.  min_tokens as in cut_at_stop_string_after."""
    if not any(stops):
        return len(tokens)
    for n in range(1, len(tokens) + 1):
        if cut_at_stop_string_after(tokenizer, tokens[:n], stops, min_tokens)[1]:
            return n
    return len(tokens)


def cut_at_stop_string_after(tokenizer, tokens, stops, min_tokens=0):
    """cut_at_stop_string of the decoded tokens: the text before the earliest-starting stop string.  With min_tokens > 0 only an
    occurrence that ends after the text of the first min_tokens tokens counts: vLLM's stop checker looks for stop strings in the new
    text of a step only once the output is longer than min_tokens, so one that completes earlier never ends the output."""
    text = decode_text(tokenizer, tokens)
    floor = len(decode_text(tokenizer, tokens[:min_tokens])) if min_tokens else 0
    starts = [i for st in stops if st for i in [text.find(st, max(0, floor - len(st) + 1))] if i >= 0]
    return (text[:min(starts)], True) if starts else (text, False)


def eos_ids(config, stop_token_ids=None, extra=None):
    """Stop ids of a request: the UNION of the model's EOS ids (config / generation_config) and the request's stop_token_ids
    (vLLM adds stop_token_ids to the EOS stop, it does not replace it; llm_utils.py:153 passes both Qwen ids explicitly)."""
    out = []
    for src in (getattr(config, "eos_token_id", None), extra, stop_token_ids):
        if src is None:
            continue
        out += [int(t) for t in (src if isinstance(src, (list, tuple, set)) else [src])]
    return sorted(set(out))


def cut_at_stop(tokens, stop_ids, ignore_eos=False):
    """(tokens before the first stop id, finish_reason).  The stop token itself is not part of the completion (vLLM strips it; the
    reference decodes with skip_special_tokens=True); whatever generate() padded a finished row with is dropped with it."""
    toks = [int(t) for t in tokens]
    if not ignore_eos:
        stop = set(int(t) for t in stop_ids)
        for i, t in enumerate(toks):
            if t in stop:
                return toks[:i], "stop"
    return toks, "length"


def engine_completion(tokenizer, r, stop_ids, ignore_eos=False, stops=(), min_tokens=0):
    """The CompletionOutput of a finished continuous-engine Request (engine.Request): the tokens before the first stop id, the text
    cut before a stop string that counts after min_tokens, the logprob dicts and cumulative_logprob of the tokens that text came
    from (when the request asked for logprobs), and the finish_reason."""
    toks, fin = cut_at_stop(r.tokens, stop_ids, ignore_eos)
    text, hit = cut_at_stop_string_after(tokenizer, toks, stops, min_tokens)
    out = CompletionOutput(text, toks, "stop" if hit else fin)
    if r.logprobs is not None:
        keep = tokens_before_stop_string(tokenizer, toks, stops, min_tokens) if hit else len(toks)
        out.logprobs = [logprob_dict(toks[j], *r.token_logprobs[j], tokenizer) for j in range(keep)]
        out.cumulative_logprob = float(sum(r.token_logprobs[j][0] for j in range(keep)))
    return out


def decode_text(tokenizer, tokens):
    """tokenizer.decode(..., skip_special_tokens=True) (inference_tsmllm_deepspeed.py:104-106), for tokenizers that take the flag."""
    try:
        return tokenizer.decode(tokens, skip_special_tokens=True)
    except TypeError:
        return tokenizer.decode(tokens)


def cut_at_stop_string(text, stops):
    cut = min([text.find(st) for st in stops if st and st in text], default=-1)
    return (text[:cut], True) if cut >= 0 else (text, False)


class IncrementalDecoder:
    """Streaming detokeniser: decodes the CUMULATIVE ids and emits only the new suffix, holding back a trailing U+FFFD (an
    incomplete multi-byte character, e.g. half of a Chinese character) until the bytes that complete it arrive."""

    def __init__(self, tokenizer):
        self.tok, self.ids, self.sent = tokenizer, [], 0

    def push(self, token_ids):
        self.ids += [int(t) for t in token_ids]
        text = decode_text(self.tok, self.ids)
        while text.endswith("\ufffd"):
            text = text[:-1]
        piece = text[self.sent:]
        self.sent = max(self.sent, len(text))
        return piece

    def flush(self):
        text = decode_text(self.tok, self.ids)
        piece = text[self.sent:]
        self.sent = len(text)
        return piece


@dataclass
class RequestOutput:
    prompt: str
    outputs: list
    num_cached_tokens: int = 0          # prompt positions (patch rows included) whose KV came from the prefix cache
    prompt_logprobs: list = None        # SamplingParams.prompt_logprobs: per prompt token, None (the first) or {id: Logprob}


def _free_port():
    import socket
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        return so.getsockname()[1]


def _tp_worker(rank, world, port, backend, factory, factory_kw):
    """Body of a spawned tensor-parallel rank (rank >= 1): join the group, build the same engine on this rank's shard, then mirror
    every call the driver (rank 0) broadcasts -- the ranks of a tensor-parallel model run the same program (SPMD)."""
    import os
    import torch.distributed as dist
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    if backend == "nccl":
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    else:
        dist.init_process_group(backend, rank=rank, world_size=world)
    engine = factory(**factory_kw)
    while True:
        box = [None]
        dist.broadcast_object_list(box, src=0)
        cmd = box[0]
        if cmd[0] == "stop":
            break
        if cmd[0] == "generate":
            engine._generate(cmd[1], cmd[2])
    dist.destroy_process_group()


def _make_llm(**kw):
    return LLM(**kw)


class LLM:
    def __init__(self, model=None, tokenizer=None, config=None, state_dict=None, tensor_parallel_size=1, dtype="bfloat16",
                 max_model_len=2048, max_num_seqs=32, limit_mm_per_prompt=None, trust_remote_code=True, seed=1234,
                 distributed_backend="nccl", quantization=None, enable_prefix_caching=False, **kw):
        """tensor_parallel_size = k > 1 (every caller of the reference passes it: demo/demo_vllm.py:30, llm_utils.py:153-154):
          * under torchrun / an initialised process group of k ranks the engine ATTACHES: every rank constructs the LLM and makes the
            same generate() calls (rank r holds shard r);
          * otherwise the constructor SPAWNS k - 1 worker processes (one per GPU, as vLLM's multiprocessing executor does,
            README.md:141) that build their shards and mirror every generate() call of this process (rank 0) -- the model must then
            be named by a path or by config + seed (a ChatTSForCausalLM instance cannot be sent to another process).
        quantization: None (the checkpoint's 16-bit weights) or "fp8" (vLLM's weight-only FP8: ChatTSForCausalLM.quantize_fp8 at load time,
        on every rank).
        enable_prefix_caching: the KV pages of a prompt prefix an earlier request wrote are reused, series included (prefix_cache.py);
        single GPU only."""
        import os
        if quantization not in (None, "fp8"):
            raise ValueError(f"quantization={quantization!r}: supported are None and 'fp8'")
        tp = int(tensor_parallel_size or 1)
        if enable_prefix_caching and tp > 1:
            raise ValueError("enable_prefix_caching is single-GPU only (tensor_parallel_size must be 1)")
        if enable_prefix_caching and isinstance(model, ChatTSForCausalLM) and not model.enable_prefix_caching:
            raise ValueError("enable_prefix_caching=True with a model built without it: construct it with enable_prefix_caching=True")
        self._tp_procs, self._tp_driver = [], False
        tp_kw = {}
        if tp > 1:
            import torch.distributed as dist
            attach = dist.is_available() and dist.is_initialized()
            if not attach and int(os.environ.get("WORLD_SIZE", "1")) == tp:          # torchrun started us: join its group
                local = int(os.environ.get("LOCAL_RANK", "0"))
                if distributed_backend == "nccl":
                    torch.cuda.set_device(local)
                    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
                else:
                    dist.init_process_group(distributed_backend)
                attach = True
            if attach:
                if dist.get_world_size() != tp:
                    raise ValueError(f"tensor_parallel_size={tp} but the process group has {dist.get_world_size()} ranks")
                tp_kw = dict(tp_rank=dist.get_rank(), tp_size=tp)
            else:
                if isinstance(model, ChatTSForCausalLM) or state_dict is not None:
                    raise ValueError("spawning tensor-parallel ranks needs a model PATH or config + seed (launch with torchrun to pass "
                                     "a constructed model or a state dict on every rank)")
                import torch.multiprocessing as mp
                port = _free_port()
                child_kw = dict(model=model, tokenizer=tokenizer, config=config, tensor_parallel_size=tp, dtype=dtype, max_model_len=max_model_len,
                                max_num_seqs=max_num_seqs, limit_mm_per_prompt=limit_mm_per_prompt, seed=seed,
                                distributed_backend=distributed_backend, quantization=quantization, **kw)
                ctx = mp.get_context("spawn")
                for r in range(1, tp):
                    pr = ctx.Process(target=_tp_worker, args=(r, tp, port, distributed_backend, _make_llm, child_kw), daemon=True)
                    pr.start()
                    self._tp_procs.append(pr)
                os.environ.update(RANK="0", LOCAL_RANK="0", WORLD_SIZE=str(tp), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
                if distributed_backend == "nccl":
                    torch.cuda.set_device(0)
                    dist.init_process_group("nccl", rank=0, world_size=tp, device_id=torch.device("cuda:0"))
                else:
                    dist.init_process_group(distributed_backend, rank=0, world_size=tp)
                self._tp_driver = True
                tp_kw = dict(tp_rank=0, tp_size=tp)
        dt = torch.bfloat16 if str(dtype) in ("bfloat16", "torch.bfloat16") else torch.float16
        if isinstance(model, ChatTSForCausalLM):
            self.model = model
        elif isinstance(model, str):
            self.model = ChatTSForCausalLM.from_pretrained(model, torch_dtype=dt, max_seq_len=max_model_len, max_batch=max_num_seqs,
                                                           quantization=quantization, enable_prefix_caching=enable_prefix_caching, **tp_kw)
        else:
            cfg = config or ChatTSConfig.chatts_14b()
            pc = dict(enable_prefix_caching=True) if enable_prefix_caching else {}
            self.model = (ChatTSForCausalLM(cfg, state_dict, dtype=dt, max_seq_len=max_model_len, max_batch=max_num_seqs, **tp_kw, **pc)
                          if state_dict is not None else
                          ChatTSForCausalLM.from_synthetic(cfg, seed=seed, dtype=dt, max_seq_len=max_model_len, max_batch=max_num_seqs, **tp_kw,
                                                           **pc))
        if quantization == "fp8" and self.model.fp8 is None:
            self.model.quantize_fp8()
        cfg = self.model.config
        self.tokenizer = tokenizer or SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id)
        self.processor = ChatTSProcessor(self.tokenizer, cfg, dtype=torch.float32)
        self.limit = (limit_mm_per_prompt or {}).get("timeseries", MAX_TS_PER_PROMPT)

    def shutdown(self):
        """Stop the spawned tensor-parallel workers (no-op otherwise)."""
        if self._tp_driver:
            import torch.distributed as dist
            dist.broadcast_object_list([("stop",)], src=0)
            for pr in self._tp_procs:
                pr.join(timeout=30)
            dist.destroy_process_group()
            self._tp_driver, self._tp_procs = False, []

    def __del__(self):
        try:
            self.shutdown()
        except Exception:  # noqa: BLE001  (interpreter teardown)
            pass

    def generate(self, inputs, sampling_params=None, use_tqdm=False, streamer=None):
        """sampling_params: one SamplingParams for every prompt, or a list of one per prompt (as vLLM takes it).  A list whose
        entries differ runs the prompts through the continuous engine (_generate_per_prompt); an all-equal list is the single
        SamplingParams."""
        if isinstance(inputs, (dict, str)):
            inputs = [inputs]
        # plain strings are text-only prompts (llm_utils.py:127 passes a list of str to the same call)
        inputs = [{"prompt": r} if isinstance(r, str) else r for r in inputs]
        if isinstance(sampling_params, (list, tuple)):
            sps = [p or SamplingParams() for p in sampling_params]
            if len(sps) != len(inputs):
                raise ValueError(f"{len(sps)} SamplingParams for {len(inputs)} prompts: give one, or one per prompt")
            if any(p != sps[0] for p in sps[1:]):
                return self._generate_per_prompt(inputs, sps, streamer)
            sampling_params = sps[0] if sps else None
        sp = sampling_params or SamplingParams()
        if (sp.logprobs is not None or sp.prompt_logprobs is not None) and self.model.tp_size > 1:
            raise ValueError("logprobs / prompt_logprobs are single-GPU only (tensor_parallel_size must be 1)")
        if sp.structured_outputs is not None and self.model.tp_size > 1:
            raise ValueError("structured_outputs are single-GPU only (tensor_parallel_size must be 1)")
        n = max(1, int(sp.n))
        if n > 1:
            # n completions per request = n copies of the request in the batch, each row with its own draw
            # (llm_utils.py:127-130 reads outputs[i].outputs[j].text for j < n)
            flat = self._generate([r for r in inputs for _ in range(n)], sp)
            return [RequestOutput(inputs[i]["prompt"], [flat[i * n + j].outputs[0] for j in range(n)], flat[i * n].num_cached_tokens,
                                  flat[i * n].prompt_logprobs) for i in range(len(inputs))]
        return self._generate(inputs, sp, streamer)

    def _generate_per_prompt(self, inputs, sps, streamer=None):
        """Prompts with different SamplingParams, through a ContinuousEngine over model.max_batch slots: each prompt keeps its own
        max_tokens, stop ids and strings, ignore_eos, n, logprobs, processors, temperature, top_k, top_p and seed.  Copy j of a
        prompt's n is drawn with seed_row = j, so a seeded prompt gets what LLM.generate([prompt], its SamplingParams) gives.
        Outputs come back in prompt order."""
        from .engine import ContinuousEngine
        if streamer is not None:
            raise ValueError("a streamer needs one SamplingParams for every prompt")
        if self.model.tp_size > 1:
            raise ValueError("per-prompt SamplingParams are single-GPU only (tensor_parallel_size must be 1)")
        for sp in sps:
            if sp.structured_outputs is not None:
                raise ValueError("structured_outputs need one SamplingParams for every prompt")
            if sp.prompt_logprobs is not None:
                raise ValueError("prompt_logprobs need one SamplingParams for every prompt")
        gd = getattr(self.model, "generation_defaults", None) or {}
        encs = []
        for req in inputs:
            ts = (req.get("multi_modal_data") or {}).get("timeseries", [])
            if len(ts) > self.limit:
                raise ValueError(f"at most {self.limit} time series per prompt")
            for t in ts:
                if not isinstance(t, (list, np.ndarray, torch.Tensor)):
                    raise TypeError(f"Unsupported time series type: {type(t)}")
            encs.append(self.processor(text=[req["prompt"]], timeseries=list(ts), padding=True, return_tensors="pt"))
        eng = ContinuousEngine(self.model)
        try:
            rids = []
            for enc, sp in zip(encs, sps):
                stop_ids = eos_ids(self.model.config, sp.stop_token_ids, gd.get("eos_token_id"))
                rep = sp.repetition_penalty if sp.repetition_penalty not in (None, 1.0) else gd.get("repetition_penalty")
                rids.append([eng.add_request(enc["input_ids"][0], enc["timeseries"], max_new_tokens=sp.max_tokens, eos_token_id=stop_ids,
                                             ignore_eos=sp.ignore_eos, logprobs=sp.logprobs, presence_penalty=sp.presence_penalty,
                                             frequency_penalty=sp.frequency_penalty, repetition_penalty=rep, logit_bias=sp.logit_bias,
                                             allowed_token_ids=sp.allowed_token_ids, min_tokens=sp.min_tokens, temperature=sp.temperature,
                                             top_k=sp.top_k if sp.top_k and sp.top_k > 0 else 0, top_p=sp.top_p, seed=sp.seed, seed_row=j)
                             for j in range(max(1, int(sp.n)))])
            done = {r.rid: r for r in eng.run()}
        finally:
            eng.close()
        outs = []
        for req, sp, ids in zip(inputs, sps, rids):
            reqs = [done[i] for i in ids]
            err = next((r.error for r in reqs if r.error is not None), None)
            if err is not None:
                raise err
            stops = [sp.stop] if isinstance(sp.stop, str) else list(sp.stop or [])
            stop_ids = eos_ids(self.model.config, sp.stop_token_ids, gd.get("eos_token_id"))
            outs.append(RequestOutput(req["prompt"], [engine_completion(self.tokenizer, r, stop_ids, sp.ignore_eos, stops, sp.min_tokens)
                                                      for r in reqs], reqs[0].cached_positions))
        return outs

    def _generate(self, inputs, sp, streamer=None):
        if self._tp_driver:                                  # the spawned ranks run the same call on their shards
            import torch.distributed as dist
            dist.broadcast_object_list([("generate", inputs, sp)], src=0)
        outs = []
        bs = self.model.max_batch
        stops = [sp.stop] if isinstance(sp.stop, str) else list(sp.stop or [])
        gd = getattr(self.model, "generation_defaults", None) or {}
        stop_ids = eos_ids(self.model.config, sp.stop_token_ids, gd.get("eos_token_id"))
        for i0 in range(0, len(inputs), bs):
            chunk = inputs[i0:i0 + bs]
            prompts, series = [], []
            for req in chunk:
                ts = (req.get("multi_modal_data") or {}).get("timeseries", [])
                if len(ts) > self.limit:
                    raise ValueError(f"at most {self.limit} time series per prompt")
                for t in ts:
                    if not isinstance(t, (list, np.ndarray, torch.Tensor)):
                        raise TypeError(f"Unsupported time series type: {type(t)}")
                prompts.append(req["prompt"])
                series.extend(ts)
            enc = self.processor(text=prompts, timeseries=series, padding=True, return_tensors="pt")
            S = enc["input_ids"].shape[1]
            ids = self.model.generate(**enc, max_new_tokens=sp.max_tokens, do_sample=sp.temperature > 0,
                                      temperature=sp.temperature, top_p=sp.top_p, top_k=(sp.top_k if sp.top_k and sp.top_k > 0 else None),
                                      ignore_eos=sp.ignore_eos, seed=(None if sp.seed is None else sp.seed + i0),
                                      eos_token_id=stop_ids, streamer=streamer,
                                      repetition_penalty=(sp.repetition_penalty if sp.repetition_penalty not in (None, 1.0) else None),
                                      logprobs=sp.logprobs, prompt_logprobs=sp.prompt_logprobs,
                                      structured_outputs=sp.structured_outputs, tokenizer=self.tokenizer,
                                      presence_penalty=sp.presence_penalty, frequency_penalty=sp.frequency_penalty, logit_bias=sp.logit_bias,
                                      allowed_token_ids=sp.allowed_token_ids, min_new_tokens=sp.min_tokens)
            res = self.model.last_logprobs if (sp.logprobs is not None or sp.prompt_logprobs is not None) else None
            for b, req in enumerate(chunk):
                # a row ends at ITS first stop id (the batch-wide tail after it is the pad fill of generate())
                toks, fin = cut_at_stop(ids[b, S:].tolist(), stop_ids, sp.ignore_eos)
                text, hit = cut_at_stop_string_after(self.tokenizer, toks, stops, sp.min_tokens)
                hits = getattr(self.model, "last_cached_positions", None)
                co = CompletionOutput(text, toks, "stop" if hit else fin)
                if sp.logprobs is not None:
                    keep = tokens_before_stop_string(self.tokenizer, toks, stops, sp.min_tokens) if hit else len(toks)
                    co.logprobs, co.cumulative_logprob = completion_logprobs(res, b, keep, toks, self.tokenizer)
                plp = prompt_logprob_dicts(res.prompt[b], self.tokenizer) if sp.prompt_logprobs is not None else None
                outs.append(RequestOutput(req["prompt"], [co], int(hits[b]) if hits is not None else 0, plp))
        return outs


# --------------------------------------------------------------------------------------------------
# Streaming surface of the reference's interactive script (chatts/utils/vllm_stream_qa.py:26-59):
#     model = AsyncLLMEngine.from_engine_args(AsyncEngineArgs(model=..., max_model_len=..., limit_mm_per_prompt={"timeseries": 15}))
#     async for request_output in model.generate(prompt, SamplingParams(max_tokens=...), request_id=...):
#         request_output.outputs[0].text            # CUMULATIVE text so far
# One request at a time per engine (the script is a chat loop); tokens come from the decode loop through the HF-streamer
# protocol of ChatTSForCausalLM.generate (put / end), one device->host read per token.
# --------------------------------------------------------------------------------------------------
@dataclass
class AsyncEngineArgs:
    model: object = None
    enforce_eager: bool = True                        # accepted and ignored: the decode step is always one CUDA graph
    gpu_memory_utilization: float = 0.9               # accepted and ignored: the KV pool is sized by max_model_len x max_num_seqs
    max_model_len: int = 2048
    tensor_parallel_size: int = 1
    limit_mm_per_prompt: dict = None
    trust_remote_code: bool = True
    dtype: str = "bfloat16"
    max_num_seqs: int = 1
    enable_prefix_caching: bool = False


class _AsyncStreamer:
    def __init__(self, loop, queue):
        self.loop, self.queue = loop, queue

    def put(self, ids):
        self.loop.call_soon_threadsafe(self.queue.put_nowait, [int(x) for x in ids.reshape(-1)[:1]])

    def end(self):
        pass


class AsyncLLMEngine:
    def __init__(self, llm):
        import threading
        self.llm = llm
        self._busy = threading.Lock()

    @classmethod
    def from_engine_args(cls, args, llm=None):
        if llm is None:
            llm = LLM(model=args.model, tensor_parallel_size=args.tensor_parallel_size, dtype=args.dtype, max_model_len=args.max_model_len,
                      max_num_seqs=args.max_num_seqs, limit_mm_per_prompt=args.limit_mm_per_prompt, trust_remote_code=args.trust_remote_code,
                      enable_prefix_caching=args.enable_prefix_caching)
        return cls(llm)

    async def generate(self, prompt, sampling_params=None, request_id=None):
        """Async generator of RequestOutput with the cumulative text (and token ids) after every new token; the last one carries the
        final text with the stop strings applied, exactly what the blocking call returns."""
        import asyncio
        loop = asyncio.get_running_loop()
        q = asyncio.Queue()
        req = {"prompt": prompt} if isinstance(prompt, str) else prompt
        sp = sampling_params or SamplingParams()
        done = object()

        def work():
            with self._busy:
                try:
                    out = self.llm.generate([req], sp, streamer=_AsyncStreamer(loop, q))[0]
                    loop.call_soon_threadsafe(q.put_nowait, (done, out))
                except BaseException as e:          # surfaced in the consumer, not lost in the worker thread
                    loop.call_soon_threadsafe(q.put_nowait, (done, e))

        fut = loop.run_in_executor(None, work)
        toks = []
        stops = [sp.stop] if isinstance(sp.stop, str) else list(sp.stop or [])
        gd = getattr(self.llm.model, "generation_defaults", None) or {}
        stop_ids = set(eos_ids(self.llm.model.config, sp.stop_token_ids, gd.get("eos_token_id")))
        ended = False
        while True:
            item = await q.get()
            if isinstance(item, tuple) and item[0] is done:
                await fut
                if isinstance(item[1], BaseException):
                    raise item[1]
                yield item[1]
                return
            if ended or (not sp.ignore_eos and any(t in stop_ids for t in item)):
                ended = True                           # the stop token and anything after it never reach the stream
                continue
            toks += item
            text = decode_text(self.llm.tokenizer, toks)
            if cut_at_stop_string_after(self.llm.tokenizer, toks, stops, sp.min_tokens)[1]:
                continue                               # the final output carries the text cut at the stop string
            if text.endswith("\ufffd"):
                continue                               # incomplete multi-byte character: wait for the bytes that complete it
            yield RequestOutput(req["prompt"], [CompletionOutput(text, list(toks))])
