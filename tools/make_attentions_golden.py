"""Generates tests/golden/attentions.pt by running the REFERENCE ITSELF (test infrastructure, like oracle/make_golden.py).

    MAGMA_REFERENCE_ROOT=<reference checkout> python tools/make_attentions_golden.py     # needs HF transformers

The reference's Magma (magma/magma.py) is built at the tiny LM size of oracle/make_golden.py with HF GPTJForCausalLM
(eager attention) standing in for its transformers fork, and add_adapters wraps its blocks: AdapterWrapper /
ParallelAdapterWrapper pass the attention probabilities through (magma/adapters.py:85-92,109-116). Its LM weights are
oracle.magma_oracle.init_weights(cfg, seed) with the weights whose names contain a key of GAINS multiplied by its
value, so the fixture stores only the seed and the gains: tests/test_attentions_cpu.py rebuilds the same weights.
Stored per variant: the inputs, the logits and `lm(inputs_embeds=x, output_attentions=True).attentions`.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import magma_oracle as O  # noqa: E402
from oracle.make_golden import TINY_LM, TINY_VIT, ClipVisualStandIn, TinyTokenizer  # noqa: E402
from oracle.ref_shims import load_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "attentions.pt")
# init_weights' scales (0.02, adapters 1e-3) give near-uniform attention rows that the adapters barely move; these
# give peaked rows, and adapters that change the second block's attentions
GAINS = {".adapter": 300.0, "q_proj": 10.0, "k_proj": 10.0}


def gained(w, gains):
    out = {}
    for k, v in w.items():
        for pat, g in gains.items():
            if pat in k:
                v = v * g
        out[k] = v
    return out


VARIANTS = {"mlp_attn_normal": {"mlp": {"adapter_type": "normal", "downsample_factor": 8},
                                "attention": {"adapter_type": "normal", "downsample_factor": 8}},
            "attn_parallel": {"attention": {"adapter_type": "parallel", "downsample_factor": 4}}}


def main():
    ref = load_reference(gptj_kwargs=TINY_LM,
                         encoder_factory=lambda name, device=None, pretrained=False: ClipVisualStandIn())
    ref.magma.get_tokenizer = lambda *a, **k: TinyTokenizer()
    ref.image_prefix.ENCODER_OUT_DIMS["clip"] = TINY_VIT["projection_dim"]
    import magma.config as mcfg

    rec = {}
    for i, (tag, ac) in enumerate(VARIANTS.items()):
        mc = mcfg.MultimodalConfig(batch_size=2, train_steps=1, encoder_name="clip", adapter_config=ac, image_seq_len=2,
                                   use_image_embed_layernorm=True, image_embed_dropout_prob=0.0, image_size=32)
        model = ref.magma.Magma(mc, device="cpu").eval()
        sd = model.state_dict()
        cfg = O.OracleConfig(d=TINY_LM["n_embd"], n_layer=TINY_LM["n_layer"], n_head=TINY_LM["n_head"],
                             rotary_dim=TINY_LM["rotary_dim"], vocab=sd["lm.lm_head.weight"].shape[0],
                             mlp_adapter=ac.get("mlp"), attn_adapter=ac.get("attention"))
        seed = 40 + i
        w = gained({k: v for k, v in O.init_weights(cfg, seed=seed, with_vit=False).items() if k.startswith("lm.")},
                   GAINS)
        lm_keys = {k for k in sd if k.startswith("lm.") and not k.endswith(("attn.bias", "masked_bias"))}
        assert set(w) == lm_keys, sorted(set(w) ^ lm_keys)
        with torch.no_grad():
            for k, v in w.items():
                sd[k].copy_(v)
        x = torch.randn(2, 12, TINY_LM["n_embd"], generator=torch.Generator().manual_seed(60 + i))
        with torch.no_grad():
            out = model.lm(inputs_embeds=x, output_attentions=True)
        assert len(out.attentions) == cfg.n_layer
        rec[tag] = {"adapter_config": ac, "seed": seed, "gains": GAINS, "lm": TINY_LM, "vocab": cfg.vocab,
                    "x": x, "logits": out.logits.clone(), "attentions": [a.clone() for a in out.attentions]}
    torch.save(rec, OUT)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
