from .agg import (Aggregation, AggregationRegistry, AttentiveAggregation, MeanAggregation, NormAggregation,
                  SumAggregation)
from .constrainer import ConstrainerFFN
from .head import (EngineBatchNorm1d, EngineBinaryClassificationFFN, EngineBinaryDirichletFFN, EngineDirichletLoss,
                   EngineEvidentialFFN, EngineEvidentialLoss, EngineLinear, EngineMPNN, EngineMulticlassClassificationFFN,
                   EngineMulticlassDirichletFFN, EngineMveFFN, EngineMVELoss, EngineQuantileFFN, EngineQuantileLoss,
                   EngineRegressionFFN)
from .message_passing import AtomMessagePassing, BondMessagePassing
from .mol_atom_bond import MABAtomMessagePassing, MABBondMessagePassing
from .transforms import GraphTransform, ScaleTransform, UnscaleTransform

__all__ = ["Aggregation", "AggregationRegistry", "AttentiveAggregation", "MeanAggregation", "NormAggregation", "SumAggregation",
           "AtomMessagePassing", "BondMessagePassing", "ConstrainerFFN", "MABAtomMessagePassing", "MABBondMessagePassing",
           "GraphTransform", "ScaleTransform", "UnscaleTransform", "EngineMPNN", "EngineRegressionFFN",
           "EngineBinaryClassificationFFN", "EngineMulticlassClassificationFFN", "EngineMveFFN", "EngineEvidentialFFN",
           "EngineQuantileFFN", "EngineBinaryDirichletFFN", "EngineMulticlassDirichletFFN", "EngineMVELoss",
           "EngineEvidentialLoss", "EngineQuantileLoss", "EngineDirichletLoss", "EngineBatchNorm1d", "EngineLinear"]
