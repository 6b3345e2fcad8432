"""Drop-in parameter containers for the reference's models.py (GraphConv, GcnEncoderGraph,
GcnEncoderNode): same constructor signatures, same parameter names / state_dict keys
(conv_first.weight, conv_block.i.weight, conv_last.weight, pred_model.weight, ...), same
initialisation (models.py:136-150), so reference checkpoints load with load_state_dict.

The explainer never calls these forwards: libgnnx's persistent kernel carries its own fused
forward/backward of exactly this architecture (models.py:58-80,230-267,363-376).  The torch
`forward` below exists for API completeness (prediction outside the explainer) and as the
plain-PyTorch fp32 statement of the op that the kernel's forward is tested against."""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn import init


class GraphConv(nn.Module):
    """models.py:9-80.  y = normalize((adj @ x) @ W + b); with att, adj is first scaled by the unnormalised attention
    (x Wa)(x Wa)^T (models.py:62-68).  The add_self variant is out of scope."""

    def __init__(self, input_dim, output_dim, add_self=False, normalize_embedding=False, dropout=0.0,
                 bias=True, gpu=True, att=False):
        super().__init__()
        if add_self:
            raise NotImplementedError("the add_self GraphConv variant is out of scope (SURVEY 8f)")
        self.att = att
        self.add_self = add_self
        self.dropout = dropout
        if dropout > 0.001:
            self.dropout_layer = nn.Dropout(p=dropout)
        self.normalize_embedding = normalize_embedding
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.weight = nn.Parameter(torch.empty(input_dim, output_dim))
        if att:
            self.att_weight = nn.Parameter(torch.empty(input_dim, input_dim))
        self.bias = nn.Parameter(torch.empty(output_dim)) if bias else None

    def forward(self, x, adj):
        if self.dropout > 0.001:
            x = self.dropout_layer(x)
        if self.att:
            x_att = torch.matmul(x, self.att_weight)
            adj = adj * (x_att @ x_att.permute(0, 2, 1))
        y = torch.matmul(torch.matmul(adj, x), self.weight)
        if self.bias is not None:
            y = y + self.bias
        if self.normalize_embedding:
            y = F.normalize(y, p=2, dim=2)
        return y, adj


class GcnEncoderGraph(nn.Module):
    """models.py:83-329 (graph classification: per-layer max-pool readout)."""

    def __init__(self, input_dim, hidden_dim, embedding_dim, label_dim, num_layers, pred_hidden_dims=[],
                 concat=True, bn=True, dropout=0.0, add_self=False, args=None):
        super().__init__()
        self.concat = concat
        self.bn = bn
        self.num_layers = num_layers
        self.num_aggs = 1
        self.bias = True if args is None else getattr(args, "bias", True)
        self.gpu = False if args is None else getattr(args, "gpu", False)
        self.att = (args is not None and getattr(args, "method", "base") == "att")
        self.conv_first = GraphConv(input_dim, hidden_dim, add_self, True, 0.0, self.bias, att=self.att)
        self.conv_block = nn.ModuleList(
            [GraphConv(hidden_dim, hidden_dim, add_self, True, dropout, self.bias, att=self.att) for _ in range(num_layers - 2)])
        self.conv_last = GraphConv(hidden_dim, embedding_dim, add_self, True, 0.0, self.bias, att=self.att)
        self.act = nn.ReLU()
        self.label_dim = label_dim
        self.pred_input_dim = hidden_dim * (num_layers - 1) + embedding_dim if concat else embedding_dim
        self.pred_model = self.build_pred_layers(self.pred_input_dim, pred_hidden_dims, label_dim)
        for m in self.modules():
            if isinstance(m, GraphConv):
                init.xavier_uniform_(m.weight.data, gain=nn.init.calculate_gain("relu"))
                if m.att:
                    init.xavier_uniform_(m.att_weight.data, gain=nn.init.calculate_gain("relu"))
                if m.bias is not None:
                    init.constant_(m.bias.data, 0.0)

    def build_pred_layers(self, in_width, hidden_widths, num_classes):
        """pred_model (models.py:193-207): a single Linear(in_width, num_classes) without hidden widths; otherwise an nn.Sequential that
        alternates Linear and the shared ReLU module and ends in a Linear to num_classes, so that the Linears sit at the even indices
        (state_dict keys pred_model.0 / .2 / ..).  Every Linear has a bias and torch's default init, drawn in the order the layers are
        listed, which is the reference's order of draws."""
        if not hidden_widths:
            return nn.Linear(in_width, num_classes)
        widths = [in_width] + list(hidden_widths)
        mods = []
        for w_in, w_out in zip(widths[:-1], widths[1:]):
            mods += [nn.Linear(w_in, w_out), self.act]
        return nn.Sequential(*mods, nn.Linear(widths[-1], num_classes))

    def apply_bn(self, x):
        bn_module = nn.BatchNorm1d(x.size()[1]).to(x.device)
        return bn_module(x)

    def _layers(self, x, adj):
        """-> (per-layer outputs, the adjacency each layer aggregated with: adj, or adj scaled by its attention)"""
        outs, adjs = [], []
        x, a = self.conv_first(x, adj)
        x = self.act(x)
        if self.bn:
            x = self.apply_bn(x)
        outs.append(x); adjs.append(a)
        for conv in self.conv_block:
            x, a = conv(x, adj)
            x = self.act(x)
            if self.bn:
                x = self.apply_bn(x)
            outs.append(x); adjs.append(a)
        x, a = self.conv_last(x, adj)
        outs.append(x); adjs.append(a)
        return outs, adjs

    def forward(self, x, adj, batch_num_nodes=None, **kwargs):
        outs, adjs = self._layers(x, adj)
        pooled = [torch.max(o, dim=1)[0] for o in outs]
        output = torch.cat(pooled, dim=1) if self.concat else pooled[-1]
        self.embedding_tensor = output
        return self.pred_model(output), torch.stack(adjs, dim=3)   # models.py:296-316

    def loss(self, pred, label, type="softmax"):
        return F.cross_entropy(pred, label)


class GcnEncoderNode(GcnEncoderGraph):
    """models.py:331-380 (node classification: Linear over the concatenated per-layer embeddings)."""

    def __init__(self, input_dim, hidden_dim, embedding_dim, label_dim, num_layers, pred_hidden_dims=[],
                 concat=True, bn=True, dropout=0.0, args=None):
        super().__init__(input_dim, hidden_dim, embedding_dim, label_dim, num_layers, pred_hidden_dims,
                         concat, bn, dropout, args=args)
        self.celoss = nn.CrossEntropyLoss()

    def forward(self, x, adj, batch_num_nodes=None, **kwargs):
        outs, adjs = self._layers(x, adj)
        self.embedding_tensor = torch.cat(outs, dim=2) if self.concat else outs[-1]
        return self.pred_model(self.embedding_tensor), torch.stack(adjs, dim=3)   # models.py:255-267

    def loss(self, pred, label):
        return self.celoss(torch.transpose(pred, 1, 2), label)
