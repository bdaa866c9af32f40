"""TEST INFRASTRUCTURE ONLY -- never imported by the product path (chemprop_b200/).

Makes the *unmodified* reference (`/root/reference`, chemprop v2.3.1) importable in this
container, where its third-party dependencies (lightning, rdkit, torchmetrics, ...) are not
installed, by registering inert ``sys.modules`` stand-ins for them.  Only the arithmetic on
the D-MPNN hot path is exercised afterwards, and that arithmetic is plain ``torch``:

* ``chemprop/nn/message_passing/base.py:135-212``  (update / finalize / forward)
* ``chemprop/nn/message_passing/mixins.py:7-30``   (initialize / message)
* ``chemprop/nn/agg.py:65-113``                    (Mean / Sum / Norm aggregation)
* ``chemprop/data/collate.py:37-62``               (BatchMolGraph collate)

``/root/reference`` does not exist on the GPU box, so nothing that runs there (`-m gpu` tests,
``smoke()``, ``bench.py``'s GPU arm) may depend on it; it is used by ``oracle/make_golden.py`` (run
here, output committed under ``tests/golden/``), by the CPU tests that pin
``oracle/restatement.py`` against the real reference when the reference tree is reachable, and by
``bench.py``'s CPU arm (``cpu_baseline`` / ``--impl reference``), which times the reference's own
modules where `reference_available()` and the oracle port otherwise, and reports which (``kind``).
"""
from __future__ import annotations

import os
import sys
import types
from unittest.mock import MagicMock

import torch
from torch import nn

REFERENCE_ROOT = os.environ.get("CHEMPROP_REFERENCE_ROOT", "/root/reference")


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "chemprop"))


def _stub(name: str, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__path__ = []
    m.__getattr__ = lambda k, _n=name: MagicMock(name=f"{_n}.{k}")
    sys.modules[name] = m
    parent, _, leaf = name.rpartition(".")
    if parent and parent in sys.modules:
        setattr(sys.modules[parent], leaf, m)
    return m


class _Names:
    """`HybridizationType.SP3` etc. -> distinct hashable values."""

    def __getattr__(self, k):
        return k


class _Metric(nn.Module):
    def __init__(self, *a, **k):
        super().__init__()

    def add_state(self, name, default, dist_reduce_fx=None):
        if isinstance(default, torch.Tensor):
            self.register_buffer(name, default)
            self.__dict__.setdefault("_state_defaults", {})[name] = default.clone()
        else:
            setattr(self, name, default)

    def forward(self, *a, **k):
        """torchmetrics.Metric.forward for `full_state_update = False` (chemprop's metrics, nn/metrics.py:62): the value of
        THIS batch -- the states are reset, updated with the batch, computed -- while the global states keep accumulating."""
        defaults = self.__dict__.get("_state_defaults", {})
        glob = {n: getattr(self, n).detach().clone() for n in defaults}
        for n, d in defaults.items():
            setattr(self, n, d.clone().to(getattr(self, n).device))
        self.update(*a, **k)
        val = self.compute()
        for n in defaults:
            setattr(self, n, glob[n] + getattr(self, n).detach())
        return val

    def clone(self):
        import copy

        return copy.deepcopy(self)


class _HyperparametersMixin:
    """Stand-in for lightning.pytorch.core.mixins.HyperparametersMixin (ctor-kwarg capture)."""

    def __init__(self, *a, **k):
        super().__init__()

    def save_hyperparameters(self, *a, ignore=(), **k):
        import inspect

        loc = inspect.currentframe().f_back.f_locals
        names = [p for p in inspect.signature(type(loc["self"]).__init__).parameters if p != "self"]
        self._hp = {n: loc[n] for n in names if n in loc and n not in ignore}

    @property
    def hparams(self):
        if not hasattr(self, "_hp"):
            self._hp = {}
        return self._hp


class _LightningModule(_HyperparametersMixin, nn.Module):
    pass


_DONE = False


def import_reference():
    """Return the imported reference package ``chemprop`` (v2.3.1)."""
    global _DONE
    if not reference_available():
        raise RuntimeError(f"reference tree not found at {REFERENCE_ROOT}")
    if not _DONE:
        for n in [
            "rdkit", "rdkit.Chem", "rdkit.Chem.rdchem", "rdkit.Chem.Descriptors",
            "rdkit.Chem.rdFingerprintGenerator", "rdkit.DataStructs", "rdkit.Chem.AllChem",
            "rdkit.Chem.rdmolops", "cuik_molmaker", "astartes", "astartes.molecules",
            "descriptastorus", "descriptastorus.descriptors",
            "descriptastorus.descriptors.rdDescriptors",
            "descriptastorus.descriptors.rdNormalizedDescriptors", "multiprocess", "myerson",
            "myerson.chemprop_explain", "myerson.chemprop_explain.utils", "configargparse",
            "torchmetrics", "torchmetrics.utilities", "torchmetrics.utilities.compute",
            "torchmetrics.utilities.data", "torchmetrics.regression", "torchmetrics.functional",
            "torchmetrics.functional.classification", "torchmetrics.classification",
        ]:
            if n not in sys.modules:
                _stub(n)
        # scaling (sklearn) and uncertainty calibration (scipy, sklearn) are imported by the package but are off the path:
        # stand-ins only where the real package is not installed
        import importlib

        for n in ["scipy", "scipy.optimize", "scipy.special", "sklearn", "sklearn.preprocessing", "sklearn.isotonic"]:
            if n not in sys.modules:
                try:
                    importlib.import_module(n)
                except ImportError:
                    _stub(n)
        sys.modules["rdkit.Chem.rdchem"].HybridizationType = _Names()
        sys.modules["rdkit.Chem.rdchem"].BondType = _Names()
        for n in ["torchmetrics", "torchmetrics.classification"]:
            for k in ["Metric", "R2Score", "BinaryAUROC", "BinaryPrecisionRecallCurve",
                      "BinaryAveragePrecision", "BinaryAccuracy", "BinaryF1Score"]:
                setattr(sys.modules[n], k, type(k, (_Metric,), {}))
        _stub("lightning", __version__="2.5.0")
        _stub("lightning.pytorch", LightningModule=_LightningModule, Trainer=MagicMock(), Callback=object)
        _stub("lightning.pytorch.core")
        _stub("lightning.pytorch.core.mixins", HyperparametersMixin=_HyperparametersMixin)
        _stub("lightning.pytorch.callbacks", Callback=object)
        _stub("lightning.pytorch.loggers")
        _stub("lightning.pytorch.strategies")
        _stub("lightning.pytorch.utilities")
        _stub("lightning.pytorch.utilities.parsing", AttributeDict=dict)
        if REFERENCE_ROOT not in sys.path:
            sys.path.insert(0, REFERENCE_ROOT)
        _DONE = True
    import chemprop  # noqa: E402

    return chemprop
