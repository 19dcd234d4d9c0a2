"""magma_b200 — Hopper-native (sm_90a) re-backing of the MAGMA forward/backward hot path.

The top-level names mirror `magma/__init__.py` of the reference (`from magma import Magma` -> `from magma_b200 import
Magma`); they resolve lazily so that `import magma_b200` (e.g. by the build script) does not pull in torch."""
__version__ = "0.1.0"

_EXPORTS = {
    "MultimodalConfig": "config", "Magma": "magma", "get_gptj": "language_model", "get_transforms": "transforms",
    "ImageInput": "image_input",
    "count_parameters": "utils", "is_main": "utils", "cycle": "utils", "get_tokenizer": "utils", "save_model": "utils",
    "load_model": "utils", "print_main": "utils", "configure_param_groups": "utils", "collate_fn": "utils",
    "build_labels": "utils", "reduce_losses": "utils",
    "eval_step": "train_loop", "train_step": "train_loop", "B200Engine": "train_loop",
    "generate": "sampling", "top_k_filter": "sampling", "top_p_filter": "sampling",
}
__all__ = sorted(_EXPORTS)


def __getattr__(name):
    mod = _EXPORTS.get(name)
    if mod is None:
        raise AttributeError(f"module 'magma_b200' has no attribute {name!r}")
    import importlib

    value = getattr(importlib.import_module(f"{__name__}.{mod}"), name)
    globals()[name] = value
    return value
