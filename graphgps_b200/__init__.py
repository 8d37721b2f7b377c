"""graphgps_b200 — H100 (sm_90a) implementation of the GraphGPS `GPSLayer` hot path.

Public surface (mirrors the reference's module boundary, SURVEY.md section 8b):
    GPSLayer      drop-in for graphgps.layer.gps_layer.GPSLayer
    GraphormerLayer  drop-in for graphgps.layer.graphormer_layer.GraphormerLayer
    BiasEncoder   drop-in for graphgps.encoder.graphormer_encoder.BiasEncoder (Graphormer's attn_bias)
    SANLayer      drop-in for graphgps.layer.san_layer.SANLayer
    SAN2Layer     drop-in for graphgps.layer.san2_layer.SAN2Layer
    GatedGCNLayer, GINEConvLayer  drop-ins for CustomGNN's graphgps.layer.gatedgcn_layer.GatedGCNLayer and
                  graphgps.layer.gine_conv_layer.GINEConvLayer
    InductiveEdgeHead  drop-in for graphgps.head.inductive_edge.GNNInductiveEdgeHead (PCQM-Contact's link head, dot
                  decoding, ranking metrics on the device)
    SANGraphHead, GraphormerHead  drop-ins for graphgps.head.san_graph.SANGraphHead and
                  graphgps.head.graphormer_graph.GraphormerHead (graph-level pooling and prediction)
    InductiveNodeHead, NodeHead, weighted_cross_entropy, cross_entropy  drop-ins for
                  graphgps.head.inductive_node.GNNInductiveNodeHead, GraphGym's GNNNodeHead and the node losses
                  (graphgps.loss.weighted_cross_entropy, GraphGym's cross_entropy), with the loss kept on the device
    KernelPENodeEncoder, rw_landing_probs  drop-in for graphgps.encoder.kernel_pos_encoder.KernelPENodeEncoder (the
                  RWSE node encoder) and the random-walk landing probabilities it reads, computed on the device
    GraphBatch    duck-typed stand-in for a collated PyG Batch (PyG is optional)
    make_batch    seeded synthetic batches of the BASELINE shapes
    GPSStack      the L-layer stack of a GPSModel (shared graph structure, plane hand-off, one gradient bucket, capture)
    GradBucket    static flat gradient storage + in-place / overlapped all-reduce (data parallel)
    BatchPrefetcher, collate   pinned pre-collated host batches, copy + graph-structure build ahead of the compute stream
"""
from .batch import GraphBatch, SHAPES, make_batch, batch_from_lists  # noqa: F401
from .gps_layer import GPSLayer  # noqa: F401
from .graphormer import GraphormerLayer  # noqa: F401
from .graphormer_bias import BiasEncoder  # noqa: F401
from .san import SAN2Layer, SANLayer  # noqa: F401
from .custom_gnn import GatedGCNLayer, GINEConvLayer  # noqa: F401
from .inductive_edge import InductiveEdgeHead  # noqa: F401
from .graph_head import GraphormerHead, SANGraphHead  # noqa: F401
from .node_head import InductiveNodeHead, NodeHead, cross_entropy, weighted_cross_entropy  # noqa: F401
from .rwse import KernelPENodeEncoder, rw_landing_probs  # noqa: F401
from .dp import GradBucket  # noqa: F401
from .stack import GPSStack  # noqa: F401
from .loader import BatchPrefetcher, collate  # noqa: F401

__all__ = ["GPSLayer", "GraphormerLayer", "BiasEncoder", "SANLayer", "SAN2Layer", "GatedGCNLayer", "GINEConvLayer", "InductiveEdgeHead", "SANGraphHead", "GraphormerHead", "InductiveNodeHead", "NodeHead",
           "weighted_cross_entropy", "cross_entropy", "KernelPENodeEncoder", "rw_landing_probs", "GPSStack", "GradBucket", "GraphBatch", "BatchPrefetcher", "collate", "SHAPES", "make_batch",
           "batch_from_lists"]
