"""TEST INFRASTRUCTURE — loads the *reference's own* Python (a checkout of Aleph-Alpha/magma whose root is given by the
environment variable MAGMA_REFERENCE_ROOT) under shims.

Only usable where that checkout exists; used by oracle/make_golden.py to pin
the CPU restatement in oracle/magma_oracle.py and to generate the committed fixtures under tests/golden/.
Nothing on the product path, in `-m gpu` tests, smoke() or bench.py imports this module.

The reference cannot be imported as-is: torchtyping, deepspeed, gdown, clip, timm are absent
and it depends on a transformers fork. The stubs below only satisfy import-time names; the arithmetic that
runs is the reference's own `magma.{adapters,image_prefix,magma,utils,sampling}` plus mainline HF GPT-J
(`transformers.models.gptj`) standing in for the fork's GPTNeo(jax=True, rotary=True) and HF CLIP-ViT standing
in for openai/CLIP's VisionTransformer.
"""
import contextlib
import os
import sys
import types

import torch
import torch.nn as nn

REFERENCE_ROOT = os.environ.get("MAGMA_REFERENCE_ROOT", "")


class _AnyType:
    def __getitem__(self, item):
        return torch.Tensor


def install_stubs():
    import transformers  # noqa: F401  (must be imported before the stubs)
    import transformers.modeling_utils as mu

    if not hasattr(mu, "no_init_weights"):
        mu.no_init_weights = contextlib.nullcontext
    tt = types.ModuleType("torchtyping")
    tt.TensorType = _AnyType()
    tt.patch_typeguard = lambda: None
    sys.modules.setdefault("torchtyping", tt)
    for name in ("deepspeed", "gdown", "timm", "wandb"):
        sys.modules.setdefault(name, types.ModuleType(name))
    clip = types.ModuleType("clip")
    clip.model = types.ModuleType("clip.model")
    clip.model.LayerNorm = nn.LayerNorm
    clip.load = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("clip is stubbed"))
    sys.modules.setdefault("clip", clip)
    sys.modules.setdefault("clip.model", clip.model)
    if not os.path.isdir(os.path.join(REFERENCE_ROOT, "magma")):
        raise RuntimeError("set MAGMA_REFERENCE_ROOT to a checkout of Aleph-Alpha/magma")
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)


class StubTokenizer:
    """id-only tokenizer: the reference only needs cls/eos ids, len() and encode/decode (utils.py:43-58)."""

    cls_token_id = 50257
    eos_token_id = 50256
    pad_token_id = 50256

    def __len__(self):
        return 50258

    def encode(self, text, return_tensors=None):
        ids = [ord(c) % 50000 for c in text]
        return torch.tensor([ids], dtype=torch.long) if return_tensors == "pt" else ids

    def decode(self, ids):
        return " ".join(str(int(i)) for i in ids)


def _bridge_attn_wrappers(magma_adapters):
    """HF >= 5 calls attn(hidden_states=...) by keyword; the reference wrappers take `x` positionally
    (adapters.py:85,109). Map the keyword onto the positional argument — no arithmetic changes."""
    for cls in (magma_adapters.AdapterWrapper, magma_adapters.ParallelAdapterWrapper):
        orig = cls.forward

        def fwd(self, x=None, *a, _orig=orig, **kw):
            if x is None:
                x = kw.pop("hidden_states")
            return _orig(self, x, *a, **kw)

        cls.forward = fwd


def load_reference(gptj_kwargs=None, encoder_factory=None, vocab=50258):
    """Import the reference package and patch its three factory seams:
    get_gptj -> HF GPTJForCausalLM, get_tokenizer -> StubTokenizer, get_image_encoder -> encoder_factory."""
    install_stubs()
    import magma.adapters as m_adapters
    import magma.image_prefix as m_prefix
    import magma.magma as m_magma
    import magma.sampling as m_sampling
    import magma.utils as m_utils
    from transformers import GPTJConfig, GPTJForCausalLM

    _bridge_attn_wrappers(m_adapters)
    kw = dict(
        vocab_size=50400, n_positions=2048, n_embd=4096, n_layer=28, n_head=16, rotary_dim=64,
        activation_function="gelu_new", resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0,
        layer_norm_epsilon=1e-5, tie_word_embeddings=False,
    )
    kw.update(gptj_kwargs or {})

    def get_gptj(**_):
        cfg = GPTJConfig(**kw)
        cfg._attn_implementation = "eager"
        return GPTJForCausalLM(cfg)

    m_magma.get_gptj = get_gptj
    m_magma.get_tokenizer = lambda *a, **k: StubTokenizer()
    if encoder_factory is not None:
        m_prefix.get_image_encoder = encoder_factory
    m_magma.get_transforms = lambda *a, **k: (lambda img: img)
    return types.SimpleNamespace(
        adapters=m_adapters, image_prefix=m_prefix, magma=m_magma, sampling=m_sampling, utils=m_utils
    )
