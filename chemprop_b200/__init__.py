"""chemprop_b200: a Hopper (H100, sm_90a) engine for chemprop's D-MPNN message-passing hot path,
behind chemprop's own module API (`nn.BondMessagePassing`, `nn.AtomMessagePassing`,
`nn.{Mean,Sum,Norm}Aggregation`, `data.BatchMolGraph`)."""
from . import data, nn  # noqa: F401
from ._lib import DmpnnError  # noqa: F401

__version__ = "0.1.0"
