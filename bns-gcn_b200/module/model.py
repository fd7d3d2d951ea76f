"""Layer stacks ``GCN`` / ``GraphSAGE`` / ``GAT`` behind the reference's constructors and ``forward`` signatures
(module/model.py:7-132).  What is an interface is kept -- class and attribute names (``layers``, ``norm``,
``dropout``: they are the state-dict keys), argument order, the order in which sub-modules are created (it fixes the
initial weights under a given seed) -- the rest is organised around one builder and one inter-layer step."""
import torch.nn.functional as F
from torch import nn

from .. import ops
from ..graph import PartitionEvalGraph
from ..helper import context as ctx
from .layer import GCNLayer, GraphSAGELayer

# LayerNorm -> ReLU -> (next layer's) dropout as one fused kernel each way (ops.LnReluDropout) when the model uses
# `--norm layer` with ReLU on CUDA; False = the three separate ATen ops of the reference (module/model.py:88-91, :80)
FUSE_NORM_ACT_DROPOUT = True


def _make_norm(kind, width, train_size):
    if kind == 'layer':
        return nn.LayerNorm(width, elementwise_affine=True)
    if kind == 'batch':
        from .sync_bn import SyncBatchNorm
        return SyncBatchNorm(width, train_size)
    return None


class GNNBase(nn.Module):

    def __init__(self, layer_size, activation, use_pp=False, dropout=0.5, norm='layer', n_linear=0):
        super().__init__()
        self.n_layers, self.n_linear = len(layer_size) - 1, n_linear
        self.activation, self.use_pp = activation, use_pp
        self.layers = nn.ModuleList()              # registered before `norm`: parameter order of the reference
        self.use_norm = norm is not None
        if self.use_norm:
            self.norm = nn.ModuleList()
        self.dropout = nn.Dropout(p=dropout)
        # fused.ParamArena, set by train.setup when the whole model can take the fused training step (fused.py);
        # None = the op-by-op autograd path
        self._arena = None
        self._scratch = None        # fused.Transient: the padded logits of the current step

    @property
    def n_conv(self) -> int:
        """Graph layers come first, ``n_linear`` plain ``nn.Linear`` layers close the stack."""
        return self.n_layers - self.n_linear

    def _populate(self, layer_size, conv, norm, train_size):
        """``conv(i, n_in, n_out)`` makes graph layer ``i``.  Layer ``i`` is created before the norm that follows it."""
        for i, (n_in, n_out) in enumerate(zip(layer_size[:-1], layer_size[1:])):
            self.layers.append(conv(i, n_in, n_out) if i < self.n_conv else nn.Linear(n_in, n_out))
            if self.use_norm and i < self.n_layers - 1:
                nm = _make_norm(norm, n_out, train_size)
                if nm is not None:
                    self.norm.append(nm)

    def _between(self, i, h, may_fuse, with_dropout=True):
        """norm -> activation after layer ``i``.  Returns ``(h, dropped)``: with ``may_fuse`` and LayerNorm + ReLU the
        fused kernel also applies the NEXT layer's input dropout (``with_dropout``; GAT drops inside its layers)."""
        nm = self.norm[i] if self.use_norm else None
        if (may_fuse and FUSE_NORM_ACT_DROPOUT and isinstance(nm, nn.LayerNorm) and self.activation is F.relu
                and nm.elementwise_affine and ops.ln_relu_dropout_supported(h, h.shape[1])):
            p = self.dropout.p if (self.training and with_dropout) else 0.0
            slots = out = None
            if self._arena is not None and self.training:
                slots = (self._arena.grad_padded(nm.weight), self._arena.grad_padded(nm.bias))
            if self.training and i + 1 < self.n_conv:
                # write straight into the head rows of the next layer's concat buffer (peer-mapped transport only)
                out = ctx.buffer.input_slot(i + 1, h.shape[0], h.shape[1])
            return ops.LnReluDropout.apply(h, nm.weight, nm.bias, nm.eps, p, ops.RNG["seed"] + 7919 * (i + 1), slots,
                                           out), True
        if nm is not None:
            h = nm(h)
        return self.activation(h), False

    def _forward(self, g, feat, *norms):
        """GCN / GraphSAGE (module/model.py:42-58, 77-93): dropout -> [exchange] -> layer -> norm -> activation."""
        h, dropped = feat, False               # dropped: this layer's input dropout was applied by the fused step
        arena = self._arena if self.training else None
        if arena is not None and self._scratch is None:
            from ..fused import Transient
            self._scratch = Transient()
        for i, layer in enumerate(self.layers):
            kw = {}
            if arena is not None and i < self.n_conv:
                # fused training step (fused.py): the layer writes its parameter gradients straight into the arena; the
                # precomputed layer 0 also applies its own input dropout (Philox, replay-safe)
                p = 0.0
                if not dropped:
                    if i == 0 and self.use_pp:
                        p = self.dropout.p
                    else:
                        h = self.dropout(h)
                kw = {"fused": (arena, p, ops.RNG["seed"] + 104729 * (i + 1), self._scratch)}
            elif not dropped:
                h = self.dropout(h)
            if i >= self.n_conv:
                h = layer(h)
            else:
                if self.training and (i > 0 or not self.use_pp):
                    h = ctx.buffer.update(i, h, overlap=True)          # model.py:47-48, 82-83
                h = layer(g, h, *norms, **kw)
            dropped = False
            if i < self.n_layers - 1:
                h, dropped = self._between(i, h, True)
        return h


class GCN(GNNBase):

    def __init__(self, layer_size, activation, use_pp, dropout=0.5, norm='layer', train_size=None, n_linear=0):
        super().__init__(layer_size, activation, use_pp, dropout, norm, n_linear)
        # only layer 0 consumes precomputed features (model.py:40)
        self._populate(layer_size, lambda i, a, b: GCNLayer(a, b, use_pp=use_pp and i == 0), norm, train_size)

    def forward(self, g, feat, in_norm=None, out_norm=None):
        return self._forward(g, feat, in_norm, out_norm)


class GraphSAGE(GNNBase):

    def __init__(self, layer_size, activation, use_pp, dropout=0.5, norm='layer', train_size=None, n_linear=0):
        super().__init__(layer_size, activation, use_pp, dropout, norm, n_linear)
        self._populate(layer_size, lambda i, a, b: GraphSAGELayer(a, b, use_pp=use_pp and i == 0), norm, train_size)   # :75

    def forward(self, g, feat, in_norm=None):
        return self._forward(g, feat, in_norm)


class GAT(GNNBase):
    """module/model.py:96-132: attention layers take the ``(source rows, destination rows)`` pair, heads are averaged,
    dropout sits inside the attention layers (and before the closing linear layers only).  ``conv`` is the attention
    layer's class, built as ``conv(in, out, heads, dropout, dropout)``: ``GATConv`` (the default) or ``GATv2Conv``
    (``--model gatv2``) or ``TransformerConv`` (``--model transformer``); ``--model graphsage-pool`` passes a
    factory of one-head ``SAGEPoolConv`` layers."""

    def __init__(self, layer_size, activation, use_pp, heads=1, dropout=0.5, norm='layer', train_size=None, n_linear=0,
                 conv=None):
        super().__init__(layer_size, activation, use_pp, dropout, norm, n_linear)
        if conv is None:
            from .gat import GATConv as conv
        self._populate(layer_size, lambda i, a, b: conv(a, b, heads, dropout, dropout), norm, train_size)
        for i, layer in enumerate(self.layers):
            layer._layer_index = i              # salts the Philox stream of the layer's attention dropout

    def forward(self, g, feat):
        h = feat
        for i, layer in enumerate(self.layers):
            if i >= self.n_conv:
                h = layer(self.dropout(h))
            elif not self.training:
                if i == 0 and self.use_pp and isinstance(g, PartitionEvalGraph):
                    h = layer(g, (h, h[0:g.n_in])).mean(1)          # layer 0 holds every halo row (train.precompute)
                else:
                    h = layer(g, h).mean(1)
            else:
                if i == 0 and self.use_pp:
                    src, dst = h, h[0:g.num_nodes('_V')]                # :120-121: layer 0 holds the stored halo rows
                else:
                    src, dst = ctx.buffer.update(i, h, overlap=True), h  # :117-118
                h = layer(g, (src, dst))
                h = h.view(h.shape[0], -1) if h.shape[1] == 1 else h.mean(1)   # the mean over one head is the head
            if i < self.n_layers - 1:
                h, _ = self._between(i, h, h.is_cuda, with_dropout=False)
        return h
