"""Run the reference's own entry scripts on smirk_b200 without modifying them.

    cd <reference checkout>;  python -m smirk_b200.dropin demo.py --input_path ... [script args]
    cd <reference checkout>;  python -m smirk_b200.dropin --train train.py configs/config_pretrain.yaml

    cd <reference checkout>;  python -m smirk_b200.dropin --train train.py configs/config_train.yaml

``--train`` (before the script) turns on the train-mode opt-in of SmirkEncoder and SmirkGenerator for the whole process
(``smirk_encoder.set_train_mode_default(True)``, one flag for both): the trainer's ``.train()`` encoder and generator
then run with batch statistics and get their weight gradients.  Without it a train-mode encoder or generator raises.

``install()`` registers our modules under the seven names the reference imports its hot-path classes
from (``demo.py:5-7,62``, ``src/smirk_trainer.py:3-6``, ``src/base_trainer.py``):

    src.smirk_encoder      -> smirk_b200.smirk_encoder    (SmirkEncoder, create_backbone, ...)
    src.FLAME.FLAME        -> smirk_b200.flame            (FLAME)
    src.renderer.renderer  -> smirk_b200.renderer         (Renderer)
    src.smirk_generator    -> smirk_b200.smirk_generator  (SmirkGenerator, ResnetBlock)
    src.losses.VGGPerceptualLoss -> smirk_b200.vgg_loss   (VGGPerceptualLoss)
    src.models.MICA.mica   -> smirk_b200.mica             (MICA; src.models.MICA.arcface stays the reference's)
    src.losses.ExpressionLoss -> smirk_b200.expression_loss (ExpressionLoss; src.losses.resnet stays the reference's)

Everything else under ``src`` (``src.FLAME.lbs``, ``src.renderer.util``, ``src.utils.*``, the other losses,
trainers) still resolves to the reference's files: the real ``src`` package is imported first and only these seven
submodules are replaced in ``sys.modules`` (and as attributes of their parent packages).
"""
import importlib
import os
import runpy
import sys
import types

_MAP = {
    "src.smirk_encoder": "smirk_b200.smirk_encoder",
    "src.FLAME.FLAME": "smirk_b200.flame",
    "src.renderer.renderer": "smirk_b200.renderer",
    "src.smirk_generator": "smirk_b200.smirk_generator",
    "src.losses.VGGPerceptualLoss": "smirk_b200.vgg_loss",
    "src.models.MICA.mica": "smirk_b200.mica",
    "src.losses.ExpressionLoss": "smirk_b200.expression_loss",
}


def _ensure_package(name, path_hint):
    """Import the reference's package if it exists on sys.path; otherwise make an empty namespace so the
    aliases still work (e.g. in tests that have no reference checkout)."""
    if name in sys.modules:
        return sys.modules[name]
    try:
        return importlib.import_module(name)
    except Exception:
        pkg = types.ModuleType(name)
        pkg.__path__ = [path_hint] if path_hint and os.path.isdir(path_hint) else []
        sys.modules[name] = pkg
        return pkg


def install(reference_root=None):
    """Alias the seven hot-path modules.  ``reference_root`` (default: cwd) is put on sys.path so the
    rest of the reference package keeps importing normally."""
    root = os.path.abspath(reference_root or os.getcwd())
    if root not in sys.path:
        sys.path.insert(0, root)
    for parent, sub in (("src", "src"), ("src.FLAME", "src/FLAME"), ("src.renderer", "src/renderer"),
                        ("src.losses", "src/losses"), ("src.models", "src/models"), ("src.models.MICA", "src/models/MICA")):
        pkg = _ensure_package(parent, os.path.join(root, sub))
        if "." in parent:
            setattr(sys.modules[parent.rsplit(".", 1)[0]], parent.rsplit(".", 1)[1], pkg)
    for ref_name, ours in _MAP.items():
        mod = importlib.import_module(ours)
        sys.modules[ref_name] = mod
        parent, leaf = ref_name.rsplit(".", 1)
        setattr(sys.modules[parent], leaf, mod)
    return sorted(_MAP)


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    train = argv[:1] == ["--train"]
    if train:
        argv = argv[1:]
    if not argv:
        raise SystemExit("usage: python -m smirk_b200.dropin [--train] <reference script.py> [script args...]")
    if train:
        from . import smirk_encoder
        smirk_encoder.set_train_mode_default(True)
    script = argv[0]
    install(os.path.dirname(os.path.abspath(script)) or os.getcwd())
    sys.argv = argv
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
