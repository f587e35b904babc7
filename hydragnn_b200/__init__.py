"""hydragnn-b200: a Blackwell-native message-passing engine behind HydraGNN's ``mpnn_type`` plugin API.

Public surface (mirrors the slice of ``hydragnn`` that sits on the per-step hot path):

    create_model, create_model_config      -- hydragnn.models.create
    Data, Batch                            -- torch_geometric.data stand-ins
    get_radius_graph[_pbc][_config]        -- hydragnn.preprocess.graph_samples_checks_and_updates
    train, validate, train_step, get_distributed_model -- hydragnn.train / hydragnn.utils.distributed
    select_optimizer, FlatSGD, FlatAdam, FlatAdamW, FlatAdamax, FlatAdagrad, FlatAdadelta, FlatRMSprop -- hydragnn.utils.optimizer
    branch_weighted_energy_forces, PaddedPredictStep -- examples/multidataset_hpo_sc26/inference_fused.py's weighted prediction
    PaddedRelaxStep                        -- examples/multidataset_hpo_sc26/structure_optimization_ASE.py's FIRE relaxation

The CUDA library is loaded lazily on first use; importing the package works on a CPU-only host.
"""
from .data import Batch, Data, collate_to_device  # noqa: F401
from .create import create_model, create_model_config, get_device, set_precision  # noqa: F401
from .radius import (get_radius_graph, get_radius_graph_config, get_radius_graph_pbc,  # noqa: F401
                     get_radius_graph_pbc_config, RadiusGraph, RadiusGraphPBC)
from .train import GraphedTrainStep, get_distributed_model, get_head_indices, train, train_step, validate  # noqa: F401

from .optim import (FlatAdadelta, FlatAdagrad, FlatAdam, FlatAdamax, FlatAdamW, FlatOptimizer, FlatRMSprop,  # noqa: F401
                    FlatSGD, select_optimizer)
from .padded import PaddedGraphStep  # noqa: F401
from .predict import PaddedPredictStep, branch_weighted_energy_forces  # noqa: F401
from .relax import PaddedRelaxStep  # noqa: F401

__version__ = "0.2.0"
