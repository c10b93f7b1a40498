"""H100-native predict()/add_examples() hot path of codelion/adaptive-classifier.

`import adaptive_classifier_b200 as adaptive_classifier` gives the public names of the reference package
(/root/reference/src/adaptive_classifier/__init__.py:1-16).  Importing needs no GPU; constructing a classifier or
calling a kernel does -- there is no CPU fallback.  Submodules are loaded on first attribute access.
"""
import importlib

__version__ = "0.1.0"

# public name -> submodule that defines it
_EXPORTS = {
    "AdaptiveClassifier": "classifier",
    "MultiLabelAdaptiveClassifier": "multilabel",
    "MultiLabelAdaptiveHead": "multilabel",
    "AdaptiveHead": "models",
    "Example": "models",
    "ModelConfig": "models",
    "PrototypeMemory": "memory",
    "FlatL2Index": "memory",
    "EWC": "ewc",
    "AdaptiveB200Error": "_cabi",
}
__all__ = sorted(_EXPORTS)


def __getattr__(name):
    sub = _EXPORTS.get(name)
    if sub is None:
        raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
    value = getattr(importlib.import_module(f"{__name__}.{sub}"), name)
    globals()[name] = value
    return value


def __dir__():
    return sorted(list(globals()) + list(_EXPORTS))
