from .agg import (Aggregation, AggregationRegistry, AttentiveAggregation, MeanAggregation, NormAggregation,
                  SumAggregation)
from .constrainer import ConstrainerFFN
from .head import (EngineBatchNorm1d, EngineBinaryClassificationFFN, EngineBinaryDirichletFFN, EngineBoundedMAE,
                   EngineBoundedMSE, EngineBoundedRMSE, EngineDirichletLoss, EngineEvidentialFFN, EngineEvidentialLoss,
                   EngineLinear, EngineMAE, EngineMPNN, EngineMulticlassClassificationFFN, EngineMulticlassDirichletFFN,
                   EngineMveFFN, EngineMVELoss, EngineNLogProbEnrichment, EnginePointQuantileLoss, EngineQuantileFFN, EngineQuantileLoss, EngineRegressionFFN, EngineRMSE,
                   EngineSID, EngineSpectralFFN, EngineWasserstein)
from .message_passing import AtomMessagePassing, BondMessagePassing
from .metrics import EngineCriterionMetric, EngineMetric, EngineMetricRegistry
from .mol_atom_bond import MABAtomMessagePassing, MABBondMessagePassing
from .mol_atom_bond_model import EngineMolAtomBondMPNN
from .multi import EngineMulticomponentMessagePassing, EngineMulticomponentMPNN
from .transforms import GraphTransform, ScaleTransform, UnscaleTransform

__all__ = ["Aggregation", "AggregationRegistry", "AttentiveAggregation", "MeanAggregation", "NormAggregation", "SumAggregation",
           "AtomMessagePassing", "BondMessagePassing", "ConstrainerFFN", "MABAtomMessagePassing", "MABBondMessagePassing",
           "GraphTransform", "ScaleTransform", "UnscaleTransform", "EngineMPNN", "EngineRegressionFFN",
           "EngineBinaryClassificationFFN", "EngineMulticlassClassificationFFN", "EngineMveFFN", "EngineEvidentialFFN",
           "EngineQuantileFFN", "EngineBinaryDirichletFFN", "EngineMulticlassDirichletFFN", "EngineMVELoss",
           "EngineEvidentialLoss", "EngineQuantileLoss", "EngineDirichletLoss", "EngineSpectralFFN", "EngineSID",
           "EngineWasserstein", "EngineMAE", "EngineRMSE", "EngineBoundedMSE", "EngineBoundedMAE", "EngineBoundedRMSE",
           "EngineBatchNorm1d", "EngineLinear", "EngineNLogProbEnrichment", "EnginePointQuantileLoss", "EngineMolAtomBondMPNN",
           "EngineMulticomponentMessagePassing", "EngineMulticomponentMPNN", "EngineMetric", "EngineMetricRegistry",
           "EngineCriterionMetric"]
