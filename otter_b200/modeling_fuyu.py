"""OtterHD / Fuyu patch path (SURVEY.md §8 a-9): `vision_embed_tokens` Linear(2700 -> hidden, with bias) on the raw
image patches and the scatter of the resulting rows into the word embeddings.

Mirrors /root/reference/src/otter_ai/models/fuyu/modeling_fuyu.py:
  * `gather_continuous_embeddings(word_embeddings, continuous_embeddings, image_patch_input_indices)` — :44-77, same
    argument names, same two `ValueError`s (batch-size mismatch :61-62, more indices than embeddings :73-76);
  * `patch_embeddings(vision_embed_tokens, image_patches)` — the list comprehension of :126-127;
  * `embed_inputs(...)` — :122-131 (word embeddings + patches, skipped when `past_key_values` is given).
The Persimmon language model itself is outside this path (SURVEY.md §8f rank 3).

Arithmetic: the wgmma GEMM with the bias in its epilogue (K = 2700 is padded to 2704 = a 16-byte row pitch inside
this module — callers pass the reference's shapes), then one scatter kernel (`otb_fuyu_scatter`) instead of the
reference's per-sample `nonzero` + indexed copy.
"""
from typing import List

import torch

from . import functional as F
from .params import f32_of

BF16 = torch.bfloat16
_wpad = {}      # id(weight) -> (version, data_ptr, padded bf16 weight)


def _padded_weight(w):
    """bf16 copy of an nn.Linear weight [N, K] with K padded to a multiple of 8 (TMA row pitch = 16 bytes)."""
    K = w.shape[1]
    Kp = (K + 7) // 8 * 8
    hit = _wpad.get(id(w))
    if hit is not None and hit[0] == w._version and hit[1] == w.data_ptr():
        return hit[2]
    wp = torch.zeros((w.shape[0], Kp), device=w.device, dtype=BF16)
    wp[:, :K] = w.detach()
    if len(_wpad) > 16:
        _wpad.clear()
    _wpad[id(w)] = (w._version, w.data_ptr(), wp)
    return wp


def patch_embeddings(vision_embed_tokens: torch.nn.Linear, image_patches) -> List[torch.Tensor]:
    """modeling_fuyu.py:126-127 — `[vision_embed_tokens(patch.to(dtype)).squeeze(0) for patch in image_patches]`.
    image_patches: tensor [b, n, K] or a list of [1, n_i, K] / [n_i, K] tensors -> list of bf16 [n_i, hidden].
    All samples go through ONE GEMM (rows concatenated); the returned tensors are row views of its output."""
    w = vision_embed_tokens.weight
    K = w.shape[1]
    rows = []
    for pt in image_patches:
        pt = pt.reshape(-1, pt.shape[-1])
        if pt.shape[-1] != K:
            raise RuntimeError(f"mat1 and mat2 shapes cannot be multiplied ({pt.shape[0]}x{pt.shape[1]} and "
                               f"{K}x{w.shape[0]})")            # what nn.Linear raises in the reference
        rows.append(pt)
    counts = [r.shape[0] for r in rows]
    wp = _padded_weight(w)
    x = torch.zeros((sum(counts), wp.shape[1]), device=w.device, dtype=BF16)
    x[:, :K] = torch.cat(rows, 0)
    bias = f32_of(vision_embed_tokens.bias) if vision_embed_tokens.bias is not None else None
    emb = F.linear_fwd(x, wp, bias=bias)
    return list(emb.split(counts, 0))


def gather_continuous_embeddings(word_embeddings: torch.Tensor, continuous_embeddings: List[torch.Tensor],
                                 image_patch_input_indices: torch.Tensor) -> torch.Tensor:
    """modeling_fuyu.py:44-77.  word_embeddings [b, s, h]; continuous_embeddings: list (len b) of [n_i, h];
    image_patch_input_indices int [b, s] (negative = keep the word embedding)."""
    if not (word_embeddings.shape[0] == len(continuous_embeddings)):
        raise ValueError(f"Batch sizes must match! Got {len(continuous_embeddings)=} and {word_embeddings.shape[0]=}")
    idx = image_patch_input_indices.to(torch.int64)
    counts = [int(c.shape[0]) for c in continuous_embeddings]
    # the reference's check, for every batch element at once (one device -> host read instead of b `nonzero` syncs)
    n_idx = (idx >= 0).sum(dim=1).tolist()
    for b, (ni, nc) in enumerate(zip(n_idx, counts)):
        if ni > nc:
            raise ValueError(f"Number of continuous embeddings continuous_embeddings[batch_idx].shape="
                             f"{tuple(continuous_embeddings[b].shape)} does not match number of continuous token ids "
                             f"src_indices.shape=({ni},) in batch element {b}.")
    mx = idx.amax(dim=1).tolist()
    for b, (m, nc) in enumerate(zip(mx, counts)):
        if m >= nc:                                  # the reference's indexed read raises here
            raise IndexError(f"index {m} is out of bounds for dimension 0 with size {nc}")
    dt = word_embeddings.dtype
    word = word_embeddings if dt == BF16 else word_embeddings.to(BF16)
    cont = torch.cat([c if c.dtype == BF16 else c.to(BF16) for c in continuous_embeddings], 0)
    off = [0]
    for c in counts:
        off.append(off[-1] + c)
    b_off = torch.tensor(off, dtype=torch.int64, device=word.device)
    out = F.fuyu_scatter(word, cont, idx, b_off)
    return out if dt == BF16 else out.to(dt)


def embed_inputs(embed_tokens: torch.nn.Module, vision_embed_tokens: torch.nn.Linear, input_ids, image_patches=None,
                 image_patches_indices=None, past_key_values=None) -> torch.Tensor:
    """modeling_fuyu.py:122-131: `inputs_embeds` of FuyuForCausalLM.forward when only `input_ids` is given."""
    inputs_embeds = embed_tokens(input_ids)
    if image_patches is not None and past_key_values is None:
        emb = patch_embeddings(vision_embed_tokens, image_patches)
        inputs_embeds = gather_continuous_embeddings(word_embeddings=inputs_embeds, continuous_embeddings=emb,
                                                     image_patch_input_indices=image_patches_indices)
    return inputs_embeds
