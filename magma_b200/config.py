"""MultimodalConfig — same field names / YAML format as the reference (magma/config.py:20-94) so the reference's
`configs/*.yml` load unchanged. The DeepSpeed-specific derived dicts of the reference (`config.py:96-137`) are
replaced by plain optimizer/scheduler fields consumed by magma_b200.train_loop.B200Engine."""
import uuid
from dataclasses import asdict, dataclass
from pathlib import Path

import yaml


def load_config(path, config_dir=Path("configs")):
    path = str(path)
    if not path.endswith(".yml"):
        path += ".yml"
    p = Path(path)
    if not p.exists():
        p = Path(config_dir) / path
    with open(p, "r") as f:
        return yaml.safe_load(f)


@dataclass
class MultimodalConfig:
    # training
    batch_size: int  # global batch (all ranks); the per-GPU batch is batch_size / world / gradient_accumulation_steps
    train_steps: int  # optimizer steps
    optimizer_name: str = "AdamW"  # only AdamW is built (train.py:96-101)
    lr: float = 8.0e-4  # peak learning rate of every group without its own
    image_enc_lr: float = None  # image encoder's own peak rate (utils.py:173-177); None = lr
    min_lr: float = 0.0  # floor of the warm-up / decay schedule
    lr_decay_iters: int = None  # None = WarmupLR (constant after warm-up), else linear decay to min_lr at this step
    gradient_accumulation_steps: int = 1  # micro-batches per optimizer step
    image_size: int = 256  # augmentation size for non-CLIP encoders (CLIP encoders use their input_resolution)
    eval_every: int = 250  # steps between eval_step calls
    eval_steps: int = 25  # batches per eval_step
    zero_stage: int = 2  # DeepSpeed ZeRO stage of the reference; unused here (flat arena + all-reduce)
    gradient_clipping: float = 1.0  # global-norm clip, folded into the fused optimizer kernel
    warmup_num_steps: int = 100  # log warm-up length
    weight_decay: float = 0.00  # AdamW decay; biases / LayerNorm / embeddings exempt (utils.py:120-146)
    run_blind: bool = False  # zero the images (train_loop.py:13-14)
    fine_tune: bool = False  # reference flag, not read on the hot path
    load_optimizer: bool = True  # restore Adam moments on resume
    # checkpointing
    save_every: int = 2500  # steps between checkpoints
    save: str = None  # checkpoint directory to write
    load: str = None  # checkpoint directory to resume from
    # data
    train_dataset_name: str = "conceptual_captions"
    eval_dataset_name: str = "/data/conceptual_captions"
    train_dataset_dir: str = "/data/coco_data"
    eval_dataset_dir: str = "/data/coco_data"
    eval_dataset_pct: float = 0.1
    # architecture
    encoder_name: str = "clip"  # clip | clip_vit_large | clip_resnet | clip_resnet_large (image_encoders.py)
    tokenizer_name: str = "gpt2"  # gpt2 + <|image|> (utils.py:43-58)
    lm_name: str = "EleutherAI/gpt-j-6B"  # GPT-J-6B architecture (language_model.py)
    image_seq_len: int = 2  # prefix tokens for pooled encoders (image_prefix.py:59-63)
    pretrained_img_encoder: bool = False  # no weight source offline; accepted for schema parity
    seq_len: int = None  # present but never read by the reference; magma_b200 uses it to set Magma.seq_len
    # freezing
    freeze_lm: bool = True  # false trains every LM parameter too (18 bytes each: ~109 GB for GPT-J-6B)
    freeze_img_encoder: bool = True  # false trains the encoder (ViT: vit_sched.cu; conv trunks: train-mode BN)
    image_embed_dropout_prob: float = 0.0  # nn.Dropout on the prefix (image_prefix.py:104)
    use_image_embed_layernorm: bool = False  # LayerNorm on the prefix (image_prefix.py:106-107)
    # adapters
    adapter_config: dict = None  # {"mlp": {...}, "attention": {...}} as consumed by Magma.add_adapters
    class_dict: dict = None  # classification head spec of the reference; unsupported here
    # logging
    name: str = None  # run name (random when None)
    log_every: int = 1  # logging cadence
    wandb_project: str = "magma"  # accepted for schema parity; nothing logs to wandb here

    def __post_init__(self):
        self.is_classifier = self.class_dict is not None
        if self.adapter_config is None:
            self.adapter_config = {}
        self.lr_scheduler = "WarmupLR" if self.lr_decay_iters is None else "WarmupDecayLR"
        if self.name is None:
            self.name = str(uuid.uuid4())[:8]

    @classmethod
    def from_yml(cls, path):
        return cls(**load_config(path))

    def to_dict(self):
        return asdict(self)

    def lr_at(self, step: int) -> float:
        """WarmupLR / WarmupDecayLR as configured for DeepSpeed in the reference (config.py:103-123):
        log-warmup to `lr` over warmup_num_steps, then constant or linear decay to min_lr at lr_decay_iters."""
        import math

        w = max(self.warmup_num_steps, 2)
        if step < w:
            gamma = math.log(step + 1) / math.log(w)
            return self.min_lr + (self.lr - self.min_lr) * gamma
        if self.lr_decay_iters is None:
            return self.lr
        frac = max(0.0, (self.lr_decay_iters - step) / max(1.0, self.lr_decay_iters - w))
        return self.min_lr + (self.lr - self.min_lr) * frac
