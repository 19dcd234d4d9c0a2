"""Checkpoint key adapter for `Magma.from_checkpoint` (magma/magma.py:278-301).

The published MAGMA checkpoint (`mp_rank_00_model_states.pt["module"]`, README.md:74) was written by the reference
with the finetuneanon/transformers GPT-Neo(jax, rotary) fork as the LM, whose parameter names differ from the HF GPT-J
names this package uses (language_model.py). The fork is not vendored, so the fork-side names below are RECALLED from
its GPT-Neo lineage, not read from source (parity unpinned): `attn.attention.{q,k,v,out}_proj`, `mlp.c_fc`,
`mlp.c_proj`, causal-mask buffers `attn.attention.{bias,masked_bias}`. Anything that does not match a rule is passed
through unchanged and reported, so a differing real checkpoint fails loudly in `load_state_dict` rather than silently.
"""
import re
from typing import Dict, List, Tuple

import torch

# (pattern, replacement) applied in order to every key
_RENAMES: List[Tuple[re.Pattern, str]] = [
    (re.compile(r"\.attention\.(q_proj|k_proj|v_proj|out_proj)\."), r".\1."),  # attn.attention.q_proj -> attn.q_proj
    (re.compile(r"\.c_fc\."), ".fc_in."),
    (re.compile(r"\.c_proj\."), ".fc_out."),
]
# non-parameter buffers of the fork's attention (causal mask, mask fill value) and learned positions (absent with rotary)
_DROP = re.compile(r"(\.attention\.(bias|masked_bias)$)|(\.attn\.(bias|masked_bias)$)|(\.transformer\.wpe\.)")


def convert_reference_state_dict(sd: Dict[str, torch.Tensor]) -> Tuple[Dict[str, torch.Tensor], Dict[str, list]]:
    """Fork-named reference state dict -> this package's names. Returns (converted, report) with
    report = {"renamed": [(old, new)], "dropped": [keys], "collisions": [keys]}."""
    out, report = {}, {"renamed": [], "dropped": [], "collisions": []}
    for k, v in sd.items():
        if not k.startswith("image_prefix.") and _DROP.search(k):
            report["dropped"].append(k)
            continue
        nk = k
        if not k.startswith("image_prefix."):  # CLIP's own ViT blocks are legitimately named mlp.c_fc / mlp.c_proj
            for pat, rep in _RENAMES:
                nk = pat.sub(rep, nk)
        if nk != k:
            report["renamed"].append((k, nk))
        if nk in out:
            report["collisions"].append(nk)
        out[nk] = v
    return out, report


def to_reference_names(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Inverse mapping (this package -> fork names), for writing checkpoints the reference can read."""
    out = {}
    for k, v in sd.items():
        nk = k
        if not k.startswith("image_prefix."):
            nk = re.sub(r"\.(attn|attn_block|module)\.(q_proj|k_proj|v_proj|out_proj)\.",
                        lambda m: f".{m.group(1)}.attention.{m.group(2)}.", k)
            nk = nk.replace(".fc_in.", ".c_fc.").replace(".fc_out.", ".c_proj.")
        out[nk] = v
    return out


# ------------------------------------------------------------------------------------------------
# Training-state checkpoints: what the reference does through the DeepSpeed engine
# (`model_engine.save_checkpoint(save_dir, client_state=sd)` / `load_checkpoint`, magma/utils.py:89-117) for
# B200Engine. Directory layout follows DeepSpeed's so `Magma.from_checkpoint` and the reference's tools find the files:
#   <save_dir>/latest                                   text file holding the tag
#   <save_dir>/<tag>/mp_rank_00_model_states.pt         {"module": state_dict, "global_step", "client_state"...}
#   <save_dir>/<tag>/b200_optim_states.pt               fp32 master / Adam moments of the flat arena + counters
# ------------------------------------------------------------------------------------------------
import os


def arena_optimizer_state(arena) -> Dict[str, object]:
    """Everything needed to resume the fused AdamW exactly: the fp32 master copy (the bf16 compute copy is derived from
    it), both moments, the step counter, and the parameter names/offsets as a layout check."""
    return {
        "names": list(arena.names), "offsets": list(arena.offsets), "numel": int(arena.numel),
        "master": arena.master.detach().cpu().clone(),
        "exp_avg": None if arena.exp_avg is None else arena.exp_avg.detach().cpu().clone(),
        "exp_avg_sq": None if arena.exp_avg_sq is None else arena.exp_avg_sq.detach().cpu().clone(),
        "step_count": int(arena.step_count),
    }


def load_arena_optimizer_state(arena, st: Dict[str, object], load_optimizer_states: bool = True) -> None:
    """Inverse of arena_optimizer_state. A layout mismatch (different trainable set / order) raises."""
    if list(st["names"]) != list(arena.names) or list(st["offsets"]) != list(arena.offsets) or \
            int(st["numel"]) != int(arena.numel):
        raise RuntimeError("optimizer checkpoint does not match the model's trainable-parameter arena "
                           f"({len(st['names'])} vs {len(arena.names)} tensors, {st['numel']} vs {arena.numel} elements)")
    arena.master.copy_(st["master"].to(arena.master.device))
    if load_optimizer_states and st["exp_avg"] is not None:
        if arena.exp_avg is None:
            arena.exp_avg = torch.zeros_like(arena.master)
            arena.exp_avg_sq = torch.zeros_like(arena.master)
        arena.exp_avg.copy_(st["exp_avg"].to(arena.master.device))
        arena.exp_avg_sq.copy_(st["exp_avg_sq"].to(arena.master.device))
        arena.step_count = int(st["step_count"])
    arena.sync_shadow(force=True)  # refresh the bf16 compute copy the kernels read


def save_training_checkpoint(save_dir, tag, module_state: Dict[str, torch.Tensor], optim_state, client_state,
                             reference_names: bool = False) -> str:
    d = os.path.join(str(save_dir), str(tag))
    os.makedirs(d, exist_ok=True)
    sd = {k: v.detach().cpu() for k, v in module_state.items()}
    if reference_names:
        sd = to_reference_names(sd)
    payload = {"module": sd}
    payload.update(client_state or {})
    torch.save(payload, os.path.join(d, "mp_rank_00_model_states.pt"))
    torch.save(optim_state, os.path.join(d, "b200_optim_states.pt"))
    with open(os.path.join(str(save_dir), "latest"), "w") as f:
        f.write(str(tag))
    return d


def read_training_checkpoint(load_dir, tag=None):
    """-> (path, model payload, optimizer state) or (None, None, None) when there is nothing to load (DeepSpeed returns
    a None path in that case and the reference's load_model then starts from step 0, magma/utils.py:112-116)."""
    latest = os.path.join(str(load_dir), "latest")
    if tag is None:
        if not os.path.exists(latest):
            return None, None, None
        tag = open(latest).read().strip()
    d = os.path.join(str(load_dir), str(tag))
    mp = os.path.join(d, "mp_rank_00_model_states.pt")
    if not os.path.exists(mp):
        return None, None, None
    payload = torch.load(mp, map_location="cpu", weights_only=False)
    op = os.path.join(d, "b200_optim_states.pt")
    optim = torch.load(op, map_location="cpu", weights_only=False) if os.path.exists(op) else None
    return d, payload, optim
