"""GraphGym-side glue for the drop-in (SURVEY.md section 8b, INTEGRATION.md section 1).

The reference instantiates ``GPSLayer`` directly in ``GPSModel.__init__`` (graphgps/network/gps_model.py:85-99,
imported at :9), so the drop-in is a rebinding of that module attribute (`install`).  GraphGym's own plugin
convention -- modules self-register with ``@register_layer(name)`` (graphgps/layer/gatedgcn_layer.py:139) -- is
served by `register`.  Neither function imports torch_geometric at module import time: this package must load
(and fail loudly on its own terms) on machines without PyG.
"""
from __future__ import annotations

import importlib

import torch

from .gps_layer import GPSLayer


def install(gps_model_module=None):
    """Rebind ``GPSLayer`` inside ``graphgps.network.gps_model`` so ``create_model()`` builds the H100 layer.

    Call after ``import graphgps`` and before ``create_model()`` (main.py:144).  Returns the class it replaced so a
    caller can restore it."""
    if gps_model_module is None:
        gps_model_module = importlib.import_module("graphgps.network.gps_model")
    previous = getattr(gps_model_module, "GPSLayer", None)
    gps_model_module.GPSLayer = GPSLayer
    return previous


def install_graphormer(graphormer_module=None):
    """Rebind ``GraphormerLayer`` inside ``graphgps.network.graphormer`` so ``GraphormerModel`` builds the H100 layer.

    Call after ``import graphgps`` and before ``create_model()``.  Returns the class it replaced so a caller can restore
    it."""
    from .graphormer import GraphormerLayer
    if graphormer_module is None:
        graphormer_module = importlib.import_module("graphgps.network.graphormer")
    previous = getattr(graphormer_module, "GraphormerLayer", None)
    graphormer_module.GraphormerLayer = GraphormerLayer
    return previous


def install_graphormer_bias(module=None):
    """Rebind ``BiasEncoder`` inside ``graphgps.encoder.graphormer_encoder`` so the ``GraphormerBias`` node encoder, and
    every composed ``*+GraphormerBias`` encoder, builds the H100 attention-bias encoder: ``GraphormerEncoder.__init__``
    looks that module global up at construction time.  Its ``NodeEncoder`` stays the reference's.

    Call after ``import graphgps`` and before ``create_model()``.  Returns the class it replaced so a caller can restore
    it."""
    from .graphormer_bias import BiasEncoder
    if module is None:
        module = importlib.import_module("graphgps.encoder.graphormer_encoder")
    previous = getattr(module, "BiasEncoder", None)
    module.BiasEncoder = BiasEncoder
    return previous


def install_san(san_module=None):
    """Rebind ``SANLayer`` inside ``graphgps.network.san_transformer`` so ``SANTransformer`` builds the H100 layer.
    ``SAN2Layer`` is left as it is (``install_san2`` rebinds it).

    Call after ``import graphgps`` and before ``create_model()``.  Returns the class it replaced so a caller can restore
    it."""
    from .san import SANLayer
    if san_module is None:
        san_module = importlib.import_module("graphgps.network.san_transformer")
    previous = getattr(san_module, "SANLayer", None)
    san_module.SANLayer = SANLayer
    return previous


def install_san2(san_module=None):
    """Rebind ``SAN2Layer`` inside ``graphgps.network.san_transformer`` so ``SANTransformer`` with
    ``cfg.gt.layer_type: SAN2Layer`` builds the H100 layer.  ``SANLayer`` is left as it is (``install_san`` rebinds it).

    Call after ``import graphgps`` and before ``create_model()``.  Returns the class it replaced so a caller can restore
    it."""
    from .san import SAN2Layer
    if san_module is None:
        san_module = importlib.import_module("graphgps.network.san_transformer")
    previous = getattr(san_module, "SAN2Layer", None)
    san_module.SAN2Layer = SAN2Layer
    return previous


def install_custom_gnn(module=None):
    """Rebind ``GatedGCNLayer`` and ``GINEConvLayer`` inside ``graphgps.network.custom_gnn`` so ``CustomGNN`` builds the
    H100 layers: ``CustomGNN.build_conv_model`` returns those module globals.

    Call after ``import graphgps`` and before ``create_model()``.  Returns the classes it replaced, as a dict by name,
    so a caller can restore them."""
    from .custom_gnn import GatedGCNLayer, GINEConvLayer
    if module is None:
        module = importlib.import_module("graphgps.network.custom_gnn")
    previous = {n: getattr(module, n, None) for n in ("GatedGCNLayer", "GINEConvLayer")}
    module.GatedGCNLayer = GatedGCNLayer
    module.GINEConvLayer = GINEConvLayer
    return previous


def install_inductive_edge_head(register_module=None):
    """Set ``register.head_dict['inductive_edge']`` to the H100 head, so GPSModel, CustomGNN and SANTransformer build it
    for ``gnn.head: inductive_edge``: each looks its head up in that registry at construction time.  The registered class
    has the reference's ``(dim_in, dim_out)`` constructor and reads ``cfg.model.edge_decoding`` and
    ``cfg.gnn.layers_post_mp`` when it is built.

    Call after ``import graphgps`` and before ``create_model()``.  Returns the class it replaced so a caller can restore
    it."""
    from .inductive_edge import InductiveEdgeHead
    if register_module is None:
        register_module = importlib.import_module("torch_geometric.graphgym.register")

    class InductiveEdgeHeadGraphGym(InductiveEdgeHead):
        """GNNInductiveEdgeHead(dim_in, dim_out) with its decoding and depth from GraphGym's cfg."""

        def __init__(self, dim_in, dim_out):
            cfg = importlib.import_module("torch_geometric.graphgym.config").cfg
            super().__init__(dim_in, dim_out, edge_decoding=cfg.model.edge_decoding,
                             layers_post_mp=cfg.gnn.layers_post_mp)

    previous = register_module.head_dict.get("inductive_edge")
    register_module.head_dict["inductive_edge"] = InductiveEdgeHeadGraphGym
    return previous


def install_graph_heads(register_module=None):
    """Set ``register.head_dict['san_graph']`` and ``['graphormer_graph']`` to the H100 heads, so GPSModel, CustomGNN,
    SANTransformer and GraphormerModel build them for ``gnn.head: san_graph`` / ``graphormer_graph``: each looks its
    head up in that registry at construction time.  The registered classes have the reference's ``(dim_in, dim_out)``
    constructor and read ``cfg.model.graph_pooling`` (and, for san_graph, ``cfg.gnn.act``) when they are built.

    Call after ``import graphgps`` and before ``create_model()``.  Returns the classes it replaced, as a dict by name,
    so a caller can restore them."""
    from .graph_head import GraphormerHead, SANGraphHead
    if register_module is None:
        register_module = importlib.import_module("torch_geometric.graphgym.register")

    def _cfg():
        return importlib.import_module("torch_geometric.graphgym.config").cfg

    class SANGraphHeadGraphGym(SANGraphHead):
        """SANGraphHead(dim_in, dim_out) with its pooling and activation from GraphGym's cfg (L = 2, as GraphGym
        builds it)."""

        def __init__(self, dim_in, dim_out):
            cfg = _cfg()
            super().__init__(dim_in, dim_out, graph_pooling=cfg.model.graph_pooling, act=cfg.gnn.act)

    class GraphormerHeadGraphGym(GraphormerHead):
        """GraphormerHead(dim_in, dim_out) with its pooling from GraphGym's cfg."""

        def __init__(self, dim_in, dim_out):
            super().__init__(dim_in, dim_out, graph_pooling=_cfg().model.graph_pooling)

    new = {"san_graph": SANGraphHeadGraphGym, "graphormer_graph": GraphormerHeadGraphGym}
    previous = {n: register_module.head_dict.get(n) for n in new}
    register_module.head_dict.update(new)
    return previous


def install_node_heads(register_module=None):
    """Set ``register.head_dict['inductive_node']`` and ``['node']`` to the H100 heads, so GPSModel, CustomGNN,
    SANTransformer and GraphormerModel build them for ``gnn.head: inductive_node`` / ``node``: each looks its head up in
    that registry at construction time.  The registered classes have the reference's ``(dim_in, dim_out)`` constructor
    and read ``cfg.gnn.layers_post_mp`` and ``cfg.gnn.dim_inner`` when they are built.

    Call after ``import graphgps`` and before ``create_model()``.  Returns the classes it replaced, as a dict by name,
    so a caller can restore them."""
    from .node_head import InductiveNodeHead, NodeHead
    if register_module is None:
        register_module = importlib.import_module("torch_geometric.graphgym.register")

    def _make(base, name):
        class NodeHeadGraphGym(base):
            """The head (dim_in, dim_out) with its MLP's depth and hidden width from GraphGym's cfg."""

            def __init__(self, dim_in, dim_out):
                cfg = importlib.import_module("torch_geometric.graphgym.config").cfg
                super().__init__(dim_in, dim_out, layers_post_mp=cfg.gnn.layers_post_mp,
                                 dim_inner=getattr(cfg.gnn, "dim_inner", None))

        NodeHeadGraphGym.__name__ = name
        return NodeHeadGraphGym

    new = {"inductive_node": _make(InductiveNodeHead, "InductiveNodeHeadGraphGym"),
           "node": _make(NodeHead, "NodeHeadGraphGym")}
    previous = {n: register_module.head_dict.get(n) for n in new}
    register_module.head_dict.update(new)
    return previous


def install_node_losses(register_module=None, train_module=None):
    """Put the node losses on the device.

    ``register.loss_dict['weighted_cross_entropy']`` becomes a function that, like the reference's, returns None unless
    ``cfg.model.loss_fun == 'weighted_cross_entropy'``.  ``graphgps.train.custom_train.compute_loss`` becomes a wrapper
    that squeezes a trailing size-1 dim as GraphGym's does and computes the multiclass ``cross_entropy`` on the device
    when ``cfg.model.loss_fun == 'cross_entropy'``, ``cfg.dataset.task_type == 'classification'``, pred is a CUDA
    float32 [M, C > 1] tensor and the labels are 1-D int64; everything else goes to the previous ``compute_loss``
    unchanged.

    Call after ``import graphgps`` and before training.  Returns what it replaced, as a dict by name
    (``weighted_cross_entropy`` and ``compute_loss``), so a caller can restore it."""
    from . import node_head
    if register_module is None:
        register_module = importlib.import_module("torch_geometric.graphgym.register")
    if train_module is None:
        train_module = importlib.import_module("graphgps.train.custom_train")

    def _cfg():
        return importlib.import_module("torch_geometric.graphgym.config").cfg

    def weighted_cross_entropy(pred, true):
        if _cfg().model.loss_fun == "weighted_cross_entropy":
            return node_head.weighted_cross_entropy(pred, true)
        return None

    previous = {"weighted_cross_entropy": register_module.loss_dict.get("weighted_cross_entropy"),
                "compute_loss": train_module.compute_loss}
    fallback = previous["compute_loss"]

    def compute_loss(pred, true):
        cfg = _cfg()
        p = pred.squeeze(-1) if pred.ndim > 1 else pred
        t = true.squeeze(-1) if true.ndim > 1 else true
        if cfg.model.loss_fun == "cross_entropy" and cfg.dataset.task_type == "classification" and p.is_cuda and \
                p.dtype == torch.float32 and p.ndim == 2 and p.shape[1] > 1 and t.ndim == 1 and t.dtype == torch.int64:
            return node_head.cross_entropy(p, t)
        return fallback(pred, true)

    register_module.loss_dict["weighted_cross_entropy"] = weighted_cross_entropy
    train_module.compute_loss = compute_loss
    return previous


_KERNEL_PE = {"RWSE": "RWSENodeEncoder", "HKdiagSE": "HKdiagSENodeEncoder", "ElstaticSE": "ElstaticSENodeEncoder"}


def install_rwse(on_device=False, kernel_module=None, register_module=None, loader_module=None):
    """Rebind ``RWSENodeEncoder``, ``HKdiagSENodeEncoder`` and ``ElstaticSENodeEncoder`` to the H100 kernel-PE encoder:
    in ``graphgps.encoder.kernel_pos_encoder``, in ``register.node_encoder_dict`` and as ``enc2_cls`` / ``enc3_cls`` of
    every composed encoder class registered there (``Atom+RWSE``, ``TypeDictNode+RWSE``, ``*+LapPE+RWSE``, ...).  Each
    keeps the reference's ``(dim_emb, expand_x=True)`` constructor and reads ``cfg.share.dim_in`` and
    ``cfg.posenc_<type>`` when it is built.

    With ``on_device=True`` the RWSE encoders also compute their statistics on the device from the batch's edges, at
    ``cfg.posenc_RWSE.kernel.times``, and ``graphgps.loader.master_loader.compute_posenc_stats`` is wrapped to drop
    ``'RWSE'`` from its ``pe_types``, so the dataset's CPU pre-transform no longer computes them.

    Call after ``import graphgps`` and before the dataset is loaded (``on_device``) and ``create_model()``.  Returns what
    it replaced, as a dict by name (``compute_posenc_stats`` too with ``on_device``), so a caller can restore it."""
    from .rwse import KernelPENodeEncoder
    if kernel_module is None:
        kernel_module = importlib.import_module("graphgps.encoder.kernel_pos_encoder")
    if register_module is None:
        register_module = importlib.import_module("torch_geometric.graphgym.register")

    def _make(kernel_type):
        class KernelPENodeEncoderGraphGym(KernelPENodeEncoder):
            """KernelPENodeEncoder(dim_emb, expand_x) with its sizes and settings from GraphGym's cfg."""

            def __init__(self, dim_emb, expand_x=True):
                cfg = importlib.import_module("torch_geometric.graphgym.config").cfg
                pecfg = getattr(cfg, f"posenc_{kernel_type}")
                times = list(pecfg.kernel.times)
                dim_pe = pecfg.dim_pe
                # without expand_x the encoder concatenates batch.x as it is: dim_emb - dim_pe columns (the width
                # composed encoders give their first encoder)
                dim_in = cfg.share.dim_in if expand_x and dim_emb > dim_pe else dim_emb - dim_pe
                super().__init__(dim_in, dim_emb, len(times), dim_pe, kernel_type=kernel_type,
                                 raw_norm_type=pecfg.raw_norm_type, model=pecfg.model, expand_x=expand_x,
                                 ksteps=times if on_device and kernel_type == "RWSE" else None,
                                 pass_as_var=pecfg.pass_as_var)

        KernelPENodeEncoderGraphGym.__name__ = _KERNEL_PE[kernel_type]
        return KernelPENodeEncoderGraphGym

    previous, swap = {}, {}
    for kernel_type, name in _KERNEL_PE.items():
        old = getattr(kernel_module, name, None)
        new = _make(kernel_type)
        previous[name] = old
        setattr(kernel_module, name, new)
        if old is not None:
            swap[old] = new
        if kernel_type in register_module.node_encoder_dict or old is not None:
            register_module.node_encoder_dict[kernel_type] = new
    for cls in list(register_module.node_encoder_dict.values()):
        for attr in ("enc2_cls", "enc3_cls"):
            enc = getattr(cls, attr, None)
            if enc is not None and enc in swap:
                setattr(cls, attr, swap[enc])
    if on_device:
        if loader_module is None:
            loader_module = importlib.import_module("graphgps.loader.master_loader")
        compute = loader_module.compute_posenc_stats
        previous["compute_posenc_stats"] = compute

        def compute_posenc_stats(data, pe_types, *args, **kwargs):
            return compute(data, [t for t in pe_types if t != "RWSE"], *args, **kwargs)

        loader_module.compute_posenc_stats = compute_posenc_stats
    return previous


def register(name="gpslayer_b200"):
    """Register a LayerConfig-style wrapper under ``name`` in GraphGym's layer registry.

    Raises ``RuntimeError`` when torch_geometric.graphgym is not importable, and (from GraphGym itself) ``KeyError``
    when the name is already taken."""
    try:
        register_mod = importlib.import_module("torch_geometric.graphgym.register")
        cfg = importlib.import_module("torch_geometric.graphgym.config").cfg
    except ImportError as e:  # pragma: no cover - depends on the host environment
        raise RuntimeError("torch_geometric.graphgym is not importable; use graphgps_b200.graphgym.install() or "
                           "construct graphgps_b200.GPSLayer directly") from e

    class GPSLayerB200GraphGym(GPSLayer):
        """dim_in == dim_out == cfg.gt.dim_hidden; layer types split as in gps_model.py:80."""

        def __init__(self, layer_config, **kwargs):
            local, glob = cfg.gt.layer_type.split("+")
            # GPSModel passes cfg.posenc_EquivStableLapPE.enable as equivstable_pe (gps_model.py:92)
            pe_cfg = getattr(cfg, "posenc_EquivStableLapPE", None)
            kwargs.setdefault("equivstable_pe", bool(pe_cfg.enable) if pe_cfg is not None else False)
            # PNA's in-degree histogram (gt_config.py:34-37; master_loader.py:226-231 fills it for PNA layer types)
            kwargs.setdefault("pna_degrees", getattr(cfg.gt, "pna_degrees", None))
            # the BigBird global model's configuration (gps_model.py:97)
            kwargs.setdefault("bigbird_cfg", getattr(cfg.gt, "bigbird", None))
            super().__init__(dim_h=layer_config.dim_out, local_gnn_type=local, global_model_type=glob,
                             num_heads=cfg.gt.n_heads, act=cfg.gnn.act, dropout=cfg.gt.dropout,
                             attn_dropout=cfg.gt.attn_dropout, layer_norm=cfg.gt.layer_norm,
                             batch_norm=cfg.gt.batch_norm, **kwargs)

    register_mod.register_layer(name, GPSLayerB200GraphGym)
    return GPSLayerB200GraphGym
