from .collate import (BatchMolGraph, Datum, MulticomponentTrainingBatch, TrainingBatch, collate_batch,
                      collate_multicomponent, tile_packing_order, tile_packing_order_of)
from .dataset import HostBatchBuffer, MulticomponentPackedDataset, PackedMolGraphDataset
from .loader import LoadedBatch, PackedBatchLoader
from .molgraph import MolGraph
from .synthetic import make_chain_graph, make_cgr_graphs, make_molecule, make_molecules

__all__ = ["BatchMolGraph", "Datum", "TrainingBatch", "collate_batch", "tile_packing_order", "tile_packing_order_of", "MolGraph", "PackedMolGraphDataset", "HostBatchBuffer",
           "MulticomponentPackedDataset", "MulticomponentTrainingBatch", "collate_multicomponent", "PackedBatchLoader", "LoadedBatch",
           "make_chain_graph", "make_cgr_graphs", "make_molecule", "make_molecules"]
