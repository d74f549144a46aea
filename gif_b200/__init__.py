"""gif_b200 -- H100-native (sm_90a) implementation of GIF's data-parallel hot path.

* ``gif_b200.model.stylegan2_common_layers`` / ``stg2_generator`` / ``stg2_discriminator``: drop-in operator and
  model classes (reference API, reference state_dict keys).
* ``gif_b200.losses``: R1 gradient penalty, path-length regulariser, logistic losses (loss_functions/losses.py).
* ``gif_b200.rasterize``: ``standard_rasterize`` / ``standard_rasterize_colors`` (+ differentiable wrapper).
* ``gif_b200.distributed``: one-process-per-GPU gradient all-reduce (replaces train.py's nn.DataParallel).
* ``install_as_reference_modules()``: makes ``from model import ...`` / ``from model.stg2_generator import ...`` in
  the reference's train.py resolve to this package.
"""
import importlib
import sys

_LAZY = ("_lib", "ops", "losses", "rasterize", "distributed", "checkpoint", "train_step", "render", "flame", "texture_space",
         "inference", "model")


def __getattr__(name):
    """Submodules load on first use: ``gif_b200.ops`` (and everything that computes) imports ``_lib``, which loads -- or
    builds with nvcc -- libgifb200.so and fails loudly without it; the host-only helpers (``gif_b200.distributed``,
    ``gif_b200.checkpoint``) stay importable on a machine with neither nvcc nor the library."""
    if name in _LAZY:
        return importlib.import_module("." + name, __name__)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")


__version__ = "0.1.0"


def install_as_reference_modules(data_parallel=True):
    """Register this package's modules under the reference's import names (``model``, ``model.stg2_generator``...).
    ``data_parallel``: also replace ``torch.nn.DataParallel`` by the one-process-per-GPU stand-in and install the
    gradient all-reduce optimiser hook (gif_b200.distributed), which is what lets train.py:344-367 run unchanged."""
    from . import model
    if data_parallel:
        from .distributed import install_data_parallel_shim
        install_data_parallel_shim()
    from .model import stg2_discriminator, stg2_generator, stylegan2_common_layers
    sys.modules["model"] = model
    sys.modules["model.stylegan2_common_layers"] = stylegan2_common_layers
    sys.modules["model.stg2_generator"] = stg2_generator
    sys.modules["model.stg2_discriminator"] = stg2_discriminator
    return model
