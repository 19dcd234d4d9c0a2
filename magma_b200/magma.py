"""Magma — same public API as magma/magma.py (`Magma(config, device)`, `forward`, `embed`, `preprocess_inputs`,
`generate`, `add_adapters`, `from_checkpoint`), assembled from the re-backed components.

Differences from the reference, all deliberate:
  * the LM is really frozen when `freeze_lm` is set (the reference only sets requires_grad=True on adapters and
    never False on anything, magma/magma.py:93-96); with `freeze_lm: false` every LM parameter trains, as in the
    reference, and any subset can be chosen with requires_grad followed by `finalize()`;
  * `seq_len` defaults to the LM's max_position_embeddings (2048) like the reference but honours `config.seq_len`
    and stays a plain attribute (`model.seq_len = 128`);
  * the word embedding is gathered straight into the fused [B,S,d] input buffer (the reference embeds the full
    padded caption and slices, magma.py:258-267) — same values;
  * trainable parameters (adapters, image_prefix.proj/ln, trainable LM weights) live in one flat fp32 arena with a
    bf16 compute copy.
"""
from copy import deepcopy
from pathlib import Path
from typing import List, Literal, Optional

import torch
import torch.nn as nn

from . import dp, ops
from .adapters import Adapter, AdapterWrapper, ParallelAdapter, ParallelAdapterWrapper
from .arena import ParamArena
from .config import MultimodalConfig
from .image_prefix import ImagePrefix
from .language_model import LMOutput, _backward_scale, get_gptj
from .sampling import generate
from .utils import build_labels, get_tokenizer, print_main


class _EmbedLMFn(torch.autograd.Function):
    """loss = LM(cat(prefix, wte[captions][:, :S-L]), labels): assembles the input in one gather kernel, runs the
    fused forward, and routes d(input)[:, :L] back to the image prefix. The logits are differentiable, and with
    want_hidden the LM's n_layer + 1 hidden states follow (loss, logits); the gradients of both join the same backward
    pass (entry 0's prefix rows included)."""

    @staticmethod
    def forward(ctx, magma, prefix, captions, labels, anchor, want_hidden=False):
        lm = magma.lm
        x = ops.embed_assemble(captions, lm.transformer.wte.compute_weight(), prefix.to(torch.bfloat16).contiguous())
        loss, logits, hidden, _ = lm._run_forward(x, labels, training=True, want_hidden=want_hidden)
        ctx.magma, ctx.generation = magma, lm._generation
        ctx.captions = captions  # row L + j of x is the embedding of captions[:, j]
        ctx.shape, ctx.L, ctx.pdtype = x.shape, prefix.shape[1], prefix.dtype
        ctx.set_materialize_grads(False)  # an output the loss does not read has no gradient to add
        return (loss, logits, *(hidden or ()))

    @staticmethod
    def backward(ctx, dloss, dlogits, *dhidden):
        lm = ctx.magma.lm
        if ctx.generation != lm._generation:
            raise RuntimeError("backward called after another training forward overwrote the saved activations")
        arena = ctx.magma._arena
        if arena is not None:
            arena._accumulate_current = arena.grads_live()
        L = ctx.L
        dx = lm._run_backward(ctx.shape, _backward_scale(lm, dloss), dhidden, (), dlogits,
                              embed=(ctx.captions[:, : ctx.shape[1] - L], L))
        if arena is not None:
            arena.publish_grads()
        dprefix = dx[:, : ctx.L, :].contiguous().to(ctx.pdtype)
        return None, dprefix, None, None, None, None


class Magma(nn.Module):
    def __init__(self, config, device=None, init_seed: Optional[int] = 0):
        super().__init__()
        if isinstance(config, (str, Path)):
            config = MultimodalConfig.from_yml(config)
        else:
            assert isinstance(config, MultimodalConfig)
        self.device = torch.device(device) if device is not None else torch.device(
            "cuda" if torch.cuda.is_available() else "cpu")
        self._require_cuda()
        self.config = config
        lm_cfg = getattr(config, "_lm_config", None)  # test hook: small architectures
        self.lm = get_gptj(config=lm_cfg, device=self.device) if lm_cfg is not None else get_gptj(device=self.device)
        self.seq_len = config.seq_len or self.lm.config.max_position_embeddings
        self.tokenizer = get_tokenizer("gpt2", sequence_length=self.seq_len)
        self.image_token = self.tokenizer.cls_token_id
        self.eos_token = self.tokenizer.eos_token_id
        n_tok = len(self.tokenizer) if lm_cfg is None else min(len(self.tokenizer), lm_cfg.vocab_size)
        self.lm.resize_token_embeddings(n_tok)
        self.lm.config.pad_token_id = self.tokenizer.eos_token_id
        self.word_embedding = self.lm.transformer.wte
        self.transformer = self.lm.transformer.h
        self.mlp_adapter_added, self.attn_adapter_added = False, False
        self.image_prefix = ImagePrefix(config=config, out_dim=self.lm.config.hidden_size, device=self.device)
        self.image_prefix_seq_len = self.image_prefix.out_seq_len
        self.transforms = None
        try:
            from .transforms import get_transforms

            self.transforms = get_transforms(config.image_size, config.encoder_name,
                                             input_resolution=self.image_prefix.enc.input_resolution)
        except Exception as e:  # torchvision / PIL preprocessing is host-side and optional
            self.transforms, self._transforms_error = None, e

        if config.adapter_config:
            mlp_config = deepcopy(config.adapter_config.get("mlp", None))
            if mlp_config:
                assert mlp_config.get("adapter_type") is not None
                self.add_adapters(location="mlp", adapter_type=mlp_config.pop("adapter_type"),
                                  downsample_factor=mlp_config.pop("downsample_factor", 4), **mlp_config)
            attn_config = deepcopy(config.adapter_config.get("attention", None))
            if attn_config:
                assert attn_config.get("adapter_type") is not None
                self.add_adapters(location="attention", adapter_type=attn_config.pop("adapter_type"), **attn_config)

        # freezing (intended semantics of magma.py:92-100)
        for name, param in self.lm.named_parameters():
            param.requires_grad = not config.freeze_lm or (bool(config.adapter_config) and "adapter" in name)
        # magma.py:98-100 freezes the encoder only when asked to (MAGMA_v1.yml trains it). The ViT family has a backward
        # pass (csrc/vit_sched.cu); the conv trunks do not (eval-mode BatchNorm folded into their weights).
        enc_trains = (not config.freeze_img_encoder) and getattr(self.image_prefix.enc, "supports_training", False)
        for param in self.image_prefix.enc.parameters():
            param.requires_grad = enc_trains
        self.encoder_trainable_requested = (not config.freeze_img_encoder) and not enc_trains
        if init_seed is not None:
            self.lm.init_weights(seed=init_seed)
            if hasattr(self.image_prefix.enc, "init_weights"):
                self.image_prefix.enc.init_weights(seed=init_seed + 1)
        self._arena = None
        self.finalize()

    def _require_cuda(self):
        if self.device.type != "cuda":
            raise RuntimeError("magma_b200 has no CPU path: construct Magma on a CUDA (sm_90) device")

    # ------------------------------------------------------------------------------------------
    def finalize(self):
        """(Re)build the trainable-parameter arena in the order gradients become ready: the LM head and ln_f, the
        blocks' adapters and weights in reverse layer order, then the word embedding and the image prefix. Call again
        after adding/removing trainable parameters (requires_grad). Raises before allocating when the arena and its Adam
        moments do not fit in the memory the device can still allocate."""
        self.lm.prepare_lm_parameters()
        named = [(n, p) for n, p in self.named_parameters() if p.requires_grad]

        named.sort(key=lambda item: dp.backward_order_key(item[0]))
        self._arena = ParamArena(named, self.device, previous=self._arena) if named else None
        self.lm.invalidate()
        self.lm.drop_training_workspace()
        self.lm.attach_arena(self._arena)
        self.image_prefix.attach_arena(self._arena)
        return self

    @property
    def arena(self):
        return self._arena

    def add_adapters(self, downsample_factor: int = 4,
                     adapter_type: Literal["normal", "parallel", "scaled_parallel"] = "normal",
                     location: Literal["mlp", "attention"] = "mlp", ff_attr: str = "mlp", attn_attr: str = "attn",
                     **adapter_kwargs):
        """magma/magma.py:102-174 — rewires `block.<ff_attr>` / `block.<attn_attr>` of every LM block in place:
        mlp + "normal" -> Sequential(mlp, Adapter); mlp + parallel forms -> ParallelAdapter(module=mlp);
        attention + "normal" -> AdapterWrapper(attn_block=attn); attention + parallel forms -> ParallelAdapterWrapper.
        The C++ runtime re-discovers the wiring from the module tree on its next call."""
        assert adapter_type in ["normal", "parallel", "scaled_parallel"], \
            "adapter_type must be one of 'normal', 'parallel', or 'scaled_parallel'"
        assert location in ["mlp", "attention"], "location must be one of 'mlp' or 'attention'"
        flag = "mlp_adapter_added" if location == "mlp" else "attn_adapter_added"
        if getattr(self, flag):
            raise ValueError("Adapter layer already added")
        width = self.lm.config.hidden_size
        is_parallel, is_scaled = adapter_type != "normal", adapter_type == "scaled_parallel"
        attr = ff_attr if location == "mlp" else attn_attr

        def on_device(mod):  # only the new adapter parameters move; the wrapped (frozen) module is already in place
            for n, p in mod.named_parameters():
                if n.startswith("adapter"):
                    p.data = p.data.to(self.device)
            return mod

        def wrap(inner):
            if location == "mlp":
                if is_parallel:
                    return on_device(ParallelAdapter(module=inner, dim=width, downsample_factor=downsample_factor,
                                                     scaled=is_scaled, **adapter_kwargs))
                return nn.Sequential(inner, on_device(Adapter(dim=width, downsample_factor=downsample_factor,
                                                              **adapter_kwargs)))
            if is_parallel:
                return on_device(ParallelAdapterWrapper(module=inner, dim=width, downsample_factor=downsample_factor,
                                                        scaled=is_scaled, **adapter_kwargs))
            return on_device(AdapterWrapper(attn_block=inner, dim=width, downsample_factor=downsample_factor,
                                            **adapter_kwargs))

        for block in self.transformer:
            setattr(block, attr, wrap(getattr(block, attr)))
        setattr(self, flag, True)
        self.lm.invalidate()

    def preprocess_inputs(self, input_list: list, embed=True) -> List[torch.Tensor]:
        """magma/magma.py:176-193."""
        from .image_input import ImageInput

        for i in range(len(input_list)):
            inp = input_list[i]
            if isinstance(inp, str):
                input_list[i] = self.tokenizer.encode(inp, return_tensors="pt")
            elif isinstance(inp, ImageInput):
                if self.transforms is None:
                    raise RuntimeError("image preprocessing is unavailable: magma_b200.transforms.get_transforms failed "
                                       f"at construction ({getattr(self, '_transforms_error', None)!r}); pass an "
                                       "already-transformed image tensor instead of an ImageInput")
                input_list[i] = inp.get_transformed_image(transform_fn=self.transforms)
            else:
                raise Exception(f"Invalid input type:{type(inp)}")
        return self.embed(input_list) if embed else input_list

    def embed(self, inputs: List[torch.Tensor]):
        """magma/magma.py:195-212 (images are forced to half precision there; bf16 here)."""
        emb_list = []
        for x in inputs:
            if x.ndim == 2:
                emb_list.append(self.word_embedding(x.to(self.device)))
            elif x.ndim == 4:
                emb_list.append(self.image_prefix(x.to(self.device).to(torch.bfloat16)))
            else:
                raise ValueError(f"Expected 2d or 4d tensor, got {x.ndim}d")
        return torch.cat(emb_list, dim=1)

    @torch.no_grad()
    def generate(self, embeddings, max_steps: int = 100, temperature: float = 0.7, top_k: int = 0, top_p: float = 0.9,
                 decode: bool = True):
        """magma/magma.py:214-236."""
        return generate(self, embeddings=embeddings, max_steps=max_steps, temperature=temperature, top_k=top_k,
                        top_p=top_p, decode=decode)

    def forward(self, images=None, captions=None, output_hidden_states: bool = False, input_embeddings=None):
        """magma/magma.py:238-276."""
        assert captions is not None, "Must provide captions in training"
        assert any([i is not None for i in [images, input_embeddings]]) and not all(
            [i is not None for i in [images, input_embeddings]]
        ), "Pass in either images, or input embeddings, not both."
        assert captions.shape[1] == self.seq_len, (
            f"in training, captions should be padded to sequence length ({self.seq_len}), "
            f"but are length {captions.shape[1]}")
        captions = captions.to(self.device).contiguous()
        if input_embeddings is None:
            if self.encoder_trainable_requested and self.training and torch.is_grad_enabled():
                raise NotImplementedError(f"freeze_img_encoder: false is not supported for the conv-trunk encoder "
                                          f"{self.config.encoder_name!r} (no backward pass); set freeze_img_encoder: true")
            input_embeddings = self.image_prefix(images)
        labels = build_labels(input_embeddings, captions, self.eos_token, self.device)
        trainable = self._arena is not None and torch.is_grad_enabled()
        if trainable:
            anchor = self._arena.params[0]
            res = _EmbedLMFn.apply(self, input_embeddings, captions, labels, anchor, output_hidden_states)
            return LMOutput(loss=res[0], logits=res[1], past_key_values=None,
                            hidden_states=tuple(res[2:]) if output_hidden_states else None)
        with torch.no_grad():
            x = ops.embed_assemble(captions, self.lm.transformer.wte.compute_weight(),
                                   input_embeddings.to(torch.bfloat16).contiguous())
        return self.lm(inputs_embeds=x, labels=labels, output_hidden_states=output_hidden_states)

    @classmethod
    def from_checkpoint(cls, config_path, checkpoint_path, device="cuda"):
        """magma/magma.py:278-301. The published checkpoint uses the fork's parameter names; checkpoint.py maps them
        onto this module's names and a mismatch raises instead of loading partially."""
        import os

        if not os.path.exists(checkpoint_path):
            raise FileNotFoundError(f"checkpoint {checkpoint_path} does not exist (no network: cannot download)")
        model = cls(config=config_path, device=device, init_seed=None)
        # weights_only=False: DeepSpeed payloads hold non-tensor client state (as checkpoint.read_training_checkpoint)
        sd = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        partial = bool(sd.get("trainable_only", False)) if isinstance(sd, dict) else False
        if "module" in sd.keys():
            sd = sd["module"]
        print_main(f"loading magma checkpoint from: {checkpoint_path}")
        from .checkpoint import convert_reference_state_dict

        sd, report = convert_reference_state_dict(sd)  # fork GPT-Neo names -> HF GPT-J names (checkpoint.py)
        missing, unexpected = model.load_state_dict(sd, strict=False)
        missing = [k for k in missing if not k.startswith(("word_embedding.", "transformer.")) and
                   not k.endswith("num_batches_tracked")]
        if partial:
            # a B200Engine.save_checkpoint(trainable_only=True) file: only what trains is in it. Loaded on top of the
            # frozen weights this constructor initialised (config paths / random init) — say so, loudly.
            frozen = {n for n, p in model.named_parameters() if not p.requires_grad}
            still = [k for k in missing if k not in frozen and k in dict(model.named_parameters())]
            if still or unexpected:
                raise RuntimeError(f"trainable-only checkpoint lacks trainable keys {still[:4]} / has unexpected keys "
                                   f"{list(unexpected)[:4]}")
            print_main(f"NOTE: {checkpoint_path} is a trainable-only checkpoint ({len(sd)} tensors); the "
                       f"{len(missing)} frozen LM / encoder tensors keep the values the config initialised. Save with "
                       "save_model(..., full=True) for a self-contained file.")
            missing = []
        if missing or unexpected:
            raise RuntimeError(f"checkpoint does not match the model: {len(missing)} missing (e.g. {missing[:4]}), "
                               f"{len(unexpected)} unexpected (e.g. {list(unexpected)[:4]}); "
                               f"{len(report['renamed'])} keys were renamed, {len(report['dropped'])} dropped")
        model.finalize()
        print_main("magma successfully loaded")
        model.eval()
        return model
