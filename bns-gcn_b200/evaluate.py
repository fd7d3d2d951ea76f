"""Evaluation + checkpoint branch of the reference's ``run`` (train.py:14-61, 308-321, 354-356, 427-456).

Off the throughput path (the reference's own benchmark runs use ``--no-eval``, README.md:110), kept so that a user of
the reference finds the same behaviour: every ``log_every`` epochs rank 0 saves ``model.state_dict()`` to
``checkpoint/<graph_name>_p<rate>_<epoch>.pth.tar``, evaluates on the full (validation) graph, appends the line to
``results/<dataset>_n<parts>_p<rate>.txt``, keeps the best model, and at the end writes ``<graph_name>_final.pth.tar``
and prints the test accuracy.  State-dict keys are the reference's parameter names (the module mirrors keep them), so
checkpoints are interchangeable.

Differences, deliberate: the reference copies the model to the CPU and evaluates in a thread pool with DGL on the host;
here the copy stays on the GPU and the full-graph forward uses the same SpMM / dense kernels as training
(``FullGraphHandle``: module/layer.py:39-45, 93-102 eval branches; GAT: ``GATConv``'s homogeneous call on the one-pass
attention kernel, module/gat.py), synchronously.

``ParallelEvaluator`` (``--parallel-eval``) splits that forward over the ranks instead: each evaluates its own nodes on
its partition with the whole halo exchanged layer by layer, and nobody builds the full graph.  Transductive runs
evaluate on the training partitions; inductive runs on partitions of their two evaluation graphs (the train | val
subgraph and the full graph, ``data.load_eval_partition``), each with its own degrees and its own precomputed layer-0
input (``eval_input``).
"""
from __future__ import annotations

import copy
import dataclasses
import os
from typing import Dict, Optional

import torch

from .data.store import eval_graph_of
from .data.synthetic import FullGraph


def calc_acc(logits: torch.Tensor, labels: torch.Tensor) -> float:
    """train.py:14-20: accuracy for single-label tasks, micro-F1 of ``logits > 0`` for multi-label ones
    (``sklearn.metrics.f1_score(labels, logits > 0, average='micro')`` = 2 TP / (2 TP + FP + FN))."""
    if labels.dim() == 1:
        if labels.shape[0] == 0:
            return 0.0
        return (logits.argmax(dim=1) == labels).sum().item() / labels.shape[0]
    pred, lab = logits > 0, labels > 0.5
    tp = (pred & lab).sum().item()
    fp = (pred & ~lab).sum().item()
    fn = (~pred & lab).sum().item()
    den = 2 * tp + fp + fn
    return 2.0 * tp / den if den else 0.0


@dataclasses.dataclass
class EvalGraph:
    """The ``val_g`` / ``test_g`` of the reference: a full homogeneous graph with its node data on the device."""
    handle: object                      # FullGraphHandle
    ndata: Dict[str, torch.Tensor]      # feat, label, train_mask, val_mask, test_mask


def build_eval_graph(fg: FullGraph, device) -> EvalGraph:
    from . import ops
    from .graph import FullGraphHandle
    dev = torch.device(device)
    a = ops.DeviceGraph.from_csr(fg.indptr.to(dev), fg.src.to(torch.int32).to(dev), fg.n_nodes)
    handle = FullGraphHandle(a, fg.in_degrees().to(dev), fg.out_degrees().to(dev))
    nd = {"feat": fg.feat.to(dev), "label": fg.label.to(dev), "train_mask": fg.train_mask.to(dev),
          "val_mask": fg.val_mask.to(dev), "test_mask": fg.test_mask.to(dev)}
    return EvalGraph(handle, nd)


def eval_graphs(fg: FullGraph, inductive: bool, device):
    """train.py:313-321: transductive -> the full graph for both; inductive -> (train | val) subgraph and the full graph
    (helper/utils.py:226-230)."""
    if not inductive:
        g = build_eval_graph(fg, device)
        return g, g
    return build_eval_graph(eval_graph_of(fg, 'val'), device), build_eval_graph(eval_graph_of(fg, 'test'), device)


def _emit(buf: str, result_file_name: Optional[str]) -> None:
    if result_file_name is not None:
        with open(result_file_name, 'a+') as f:
            f.write(buf + '\n')
    print(buf)


@torch.no_grad()
def evaluate_induc(name, model, g: EvalGraph, mode, result_file_name=None):
    """train.py:22-41.  ``mode``: 'val' or 'test'."""
    model.eval()
    feat, labels = g.ndata['feat'], g.ndata['label']
    mask = g.ndata[mode + '_mask']
    logits = model(g.handle, feat)
    acc = calc_acc(logits[mask], labels[mask])
    _emit("{:s} | Accuracy {:.2%}".format(name, acc), result_file_name)
    return model, acc


@torch.no_grad()
def evaluate_trans(name, model, g: EvalGraph, result_file_name=None):
    """train.py:44-61."""
    model.eval()
    feat, labels = g.ndata['feat'], g.ndata['label']
    val_mask, test_mask = g.ndata['val_mask'], g.ndata['test_mask']
    logits = model(g.handle, feat)
    val_acc = calc_acc(logits[val_mask], labels[val_mask])
    test_acc = calc_acc(logits[test_mask], labels[test_mask])
    _emit("{:s} | Validation Accuracy {:.2%} | Test Accuracy {:.2%}".format(name, val_acc, test_acc), result_file_name)
    return model, val_acc


def result_file_name(args) -> str:
    """train.py:356."""
    return 'results/%s_n%d_p%.2f.txt' % (args.dataset, args.n_partitions, args.sampling_rate)


def checkpoint_path(args, epoch: Optional[int] = None) -> str:
    """train.py:428 (periodic) and :452 (final)."""
    if epoch is None:
        return 'checkpoint/' + args.graph_name + '_final.pth.tar'
    return 'checkpoint/%s_p%.2f_%d.pth.tar' % (args.graph_name, args.sampling_rate, epoch)


def save_checkpoint(model: torch.nn.Module, path: str) -> None:
    os.makedirs(os.path.dirname(path) or '.', exist_ok=True)
    torch.save({k: v.detach().cpu() for k, v in model.state_dict().items()}, path)


def load_checkpoint(model: torch.nn.Module, path: str, strict: bool = True):
    """Load a checkpoint written by this build or by the reference (same keys, same shapes)."""
    return model.load_state_dict(torch.load(path, map_location='cpu'), strict=strict)


class Evaluator:
    """Rank 0's bookkeeping of train.py:354-356, 427-456."""

    def __init__(self, args, fg: FullGraph, device):
        self.args = args
        os.makedirs('checkpoint/', exist_ok=True)            # train.py:310-311
        os.makedirs('results/', exist_ok=True)
        self.val_g, self.test_g = eval_graphs(fg, args.inductive, device)
        self.best_model, self.best_acc = None, 0.0
        self.result_file_name = result_file_name(args)

    def after_epoch(self, model: torch.nn.Module, epoch: int) -> float:
        """train.py:427-442 at an epoch with ``(epoch + 1) % log_every == 0``."""
        save_checkpoint(model, checkpoint_path(self.args, epoch))
        snap = copy.deepcopy(model)
        was_training = model.training
        if not self.args.inductive:
            _, val_acc = evaluate_trans('Epoch %05d' % epoch, snap, self.val_g, self.result_file_name)
        else:
            _, val_acc = evaluate_induc('Epoch %05d' % epoch, snap, self.val_g, 'val', self.result_file_name)
        if val_acc > self.best_acc or self.best_model is None:
            self.best_acc, self.best_model = val_acc, snap
        model.train(was_training)
        return val_acc

    def finish(self, model: torch.nn.Module) -> float:
        """train.py:446-456."""
        if self.best_model is None:
            self.best_model = copy.deepcopy(model)
        save_checkpoint(self.best_model, checkpoint_path(self.args))
        print('model saved')
        print("Max Validation Accuracy {:.2%}".format(self.best_acc))
        _, acc = evaluate_induc('Test Result', self.best_model, self.test_g, 'test')
        return acc


def acc_counts(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """What ``calc_acc`` needs, as sums that add up across ranks: ``[correct, total]`` for single-label tasks,
    ``[TP, FP, FN]`` of ``logits > 0`` for multi-label ones (float64 on the device: exact up to 2^53)."""
    if labels.dim() == 1:
        correct = (logits.argmax(dim=1) == labels).sum()
        return torch.stack([correct, correct.new_tensor(labels.shape[0])]).double()
    pred, lab = logits > 0, labels > 0.5
    return torch.stack([(pred & lab).sum(), (pred & ~lab).sum(), (~pred & lab).sum()]).double()


def acc_of_counts(c: torch.Tensor) -> float:
    """``calc_acc`` from the summed counts of ``acc_counts``."""
    c = c.tolist()
    if len(c) == 2:
        return c[0] / c[1] if c[1] else 0.0
    den = 2 * c[0] + c[1] + c[2]
    return 2.0 * c[0] / den if den else 0.0


def _partition_eval_graph(a_in, a_out, node_dict, boundary, comm):
    from .graph import PartitionEvalGraph
    from .train import _halo_counts, collect_out_degree
    dev = a_in.device
    nd = {k: node_dict[k].to(dev) for k in ('part_id', 'in_deg', 'out_deg')}
    out_deg = collect_out_degree(nd, boundary)
    return PartitionEvalGraph(a_in, a_out, _halo_counts(nd), boundary, nd['in_deg'], out_deg, comm)


def build_partition_eval_graph(part, node_dict, boundary, comm):
    """``graph.PartitionEvalGraph`` of a training partition (``train.setup``'s ``part`` and ``boundary``; ``node_dict``
    of ``load_partition``).  Collective: the halo's out-degrees come from their owners (``train.collect_out_degree``)."""
    return _partition_eval_graph(part.a_in, part.a_out, node_dict, boundary, comm)


def eval_input(args, g, feat: torch.Tensor) -> torch.Tensor:
    """Layer 0's input on the evaluation partition ``g`` (a ``PartitionEvalGraph``) from its inner rows' raw features,
    what ``train.precompute`` gives a training partition: under ``--use-pp`` GraphSAGE's ``[x | mean over the
    in-neighbours]`` and GCN's ``D_in^-1/2 A D_out^-1/2 x`` over the inner rows; GAT (its layer 0 always takes the
    stored rows, ``train.create_model``) the inner rows followed by every halo row.  Degrees are those of ``g``'s own
    graph; the halo rows come through ``g``'s exchange (collective)."""
    from .train import ATTENTION_STACK
    if not (args.use_pp or args.model in ATTENTION_STACK):
        return feat
    n_in, n_feat = feat.shape
    with torch.no_grad():
        if args.model in ATTENTION_STACK:
            h = torch.empty(n_in + g.n_halo, n_feat, dtype=feat.dtype, device=feat.device)
            h[:n_in] = feat
            for j, _, xr in g.peer_rows(feat.contiguous()):
                b0 = n_in + g.halo_begin[j]
                h[b0:b0 + g.halo_count[j]] = xr
            return h
        pad = (-n_feat) % 4                       # 16-byte vector path of the SpMM (602 -> 604 columns)
        x = torch.nn.functional.pad(feat, (0, pad)) if pad else feat.contiguous()
        if args.model == 'graphsage':
            mean = g.aggregate(x, 1.0 / g.in_degrees().float())
            return torch.cat([feat, mean[:, :n_feat]], dim=1)
        if args.model == 'gcn':
            h = g.aggregate(x, 1.0 / torch.sqrt(g.in_degrees().float()), 1.0 / torch.sqrt(g.out_degrees().float()))
            return h[:, :n_feat].contiguous()
    raise NotImplementedError(args.model)


@dataclasses.dataclass
class EvalPart:
    """One rank's share of an evaluation graph, ready for the forward."""
    graph: object                       # graph.PartitionEvalGraph
    feat: torch.Tensor                  # layer 0's input (``eval_input``)
    labels: torch.Tensor
    mask: torch.Tensor                  # the nodes it is scored on


def build_eval_part(args, part, which: str, device, comm) -> EvalPart:
    """``EvalPart`` of ``part`` = ``(subg, node_dict, gpb)`` of ``data.load_eval_partition(args, which, rank)``:
    ``a_in`` / ``a_out`` (``train.get_in_out_graph``), the boundary (``get_boundary``), the halo's out-degrees
    (``train.collect_out_degree``) and layer 0's input -- no training buffer, no sampler.  Collective."""
    from .data.partition import NID
    from .helper.utils import get_boundary
    from .train import get_in_out_graph
    subg, node_dict, gpb = part
    dev = torch.device(device)
    nd = {k: v.to(dev) for k, v in node_dict.items()}
    a_in, a_out = get_in_out_graph(subg, nd, dev, getattr(args, 'chunk_nnz', 0))
    boundary = get_boundary({k: nd[k] for k in ('part_id', NID)}, gpb)
    g = _partition_eval_graph(a_in, a_out, nd, boundary, comm)
    return EvalPart(g, eval_input(args, g, nd['feat']), nd['label'], nd[which + '_mask'])


class ParallelEvaluator:
    """``Evaluator`` with the evaluation forward split over the ranks (``--parallel-eval``): each rank computes the
    logits of its own inner nodes on its partition with every halo node present (``graph.PartitionEvalGraph``: the
    whole boundary exchanged layer by layer), counts its masked nodes, and the counts are summed over the ranks --
    every rank gets the same accuracy.  No rank builds the whole graph.

    Transductive runs evaluate on the training partition (``graph``, ``feat`` its layer-0 input).  Inductive runs
    (``ParallelEvaluator.inductive``) evaluate on partitions of their own evaluation graphs, as ``Evaluator`` does on
    the whole ones: ``val_mask`` on the train | val subgraph after each logged epoch, ``test_mask`` on the full graph at
    ``finish`` -- whose partition is built only then (``test_part``), after the val graph's is released.

    Collective: ALL ranks call ``after_epoch`` / ``finish`` at the same epochs.  Rank 0 alone writes the checkpoints and
    the result lines (same names and formats as ``Evaluator``); every rank keeps its own snapshot of the best model (the
    weights are replicated), so the final test pass needs no broadcast."""

    def __init__(self, args, graph, feat: torch.Tensor, labels: torch.Tensor, val_mask: torch.Tensor,
                 test_mask: Optional[torch.Tensor], comm, test_part=None):
        self.args, self.graph, self.comm = args, graph, comm
        self.feat, self.labels, self.val_mask, self.test_mask = feat, labels, val_mask, test_mask
        self.test_part, self.inductive = test_part, test_part is not None
        self.is_root = comm.rank == 0
        if self.is_root:
            os.makedirs('checkpoint/', exist_ok=True)
            os.makedirs('results/', exist_ok=True)
        self.best_model, self.best_acc = None, 0.0
        self.result_file_name = result_file_name(args)

    @classmethod
    def inductive_from_parts(cls, args, eval_parts, device, comm) -> "ParallelEvaluator":
        """``--parallel-eval --inductive``: ``eval_parts = {'val': part, 'test': part}``, this rank's parts of the two
        evaluation graphs as ``data.load_eval_partition`` returns them.  Builds the val graph's ``EvalPart`` now."""
        v = build_eval_part(args, eval_parts['val'], 'val', device, comm)
        return cls(args, v.graph, v.feat, v.labels, v.mask, None, comm, test_part=eval_parts['test'])

    @torch.no_grad()
    def logits(self, model: torch.nn.Module) -> torch.Tensor:
        """This rank's inner nodes' logits (collective)."""
        model.eval()
        return model(self.graph, self.feat)

    def _acc(self, logits: torch.Tensor, mask: torch.Tensor) -> float:
        c = acc_counts(logits[mask], self.labels[mask])
        self.comm.all_reduce_sum(c)
        return acc_of_counts(c)

    def after_epoch(self, model: torch.nn.Module, epoch: int) -> float:
        if self.is_root:
            save_checkpoint(model, checkpoint_path(self.args, epoch))
        snap = copy.deepcopy(model)
        was_training = model.training
        logits = self.logits(snap)
        if self.inductive:
            val_acc = self._acc(logits, self.val_mask)
            if self.is_root:
                _emit("{:s} | Accuracy {:.2%}".format('Epoch %05d' % epoch, val_acc), self.result_file_name)
        else:
            val_acc, test_acc = self._acc(logits, self.val_mask), self._acc(logits, self.test_mask)
            if self.is_root:
                _emit("{:s} | Validation Accuracy {:.2%} | Test Accuracy {:.2%}".format('Epoch %05d' % epoch, val_acc,
                                                                                         test_acc), self.result_file_name)
        if val_acc > self.best_acc or self.best_model is None:
            self.best_acc, self.best_model = val_acc, snap
        model.train(was_training)
        return val_acc

    def use_test_graph(self) -> None:
        """Inductive: release the val graph and build this rank's part of the test graph in its place (collective;
        ``finish`` calls it, a no-op when it already ran or the run is transductive)."""
        if self.test_part is None:
            return
        dev = self.feat.device
        self.graph = self.feat = self.labels = self.val_mask = None
        t = build_eval_part(self.args, self.test_part, 'test', dev, self.comm)
        self.graph, self.feat, self.labels, self.test_mask = t.graph, t.feat, t.labels, t.mask
        self.test_part = None

    def finish(self, model: torch.nn.Module) -> float:
        if self.best_model is None:
            self.best_model = copy.deepcopy(model)
        if self.is_root:
            save_checkpoint(self.best_model, checkpoint_path(self.args))
            print('model saved')
            print("Max Validation Accuracy {:.2%}".format(self.best_acc))
        self.use_test_graph()
        acc = self._acc(self.logits(self.best_model), self.test_mask)
        if self.is_root:
            _emit("{:s} | Accuracy {:.2%}".format('Test Result', acc), None)
        return acc
