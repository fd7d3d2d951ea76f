"""The training state behind ``--save-state-every`` / ``--resume``: what a stopped run needs to continue exactly where
it stopped.

The reference saves the model's ``state_dict`` alone (train.py:428, :452) and cannot resume.  Here everything else that
changes from one epoch to the next is a function of the epoch index and the seed -- the boundary sampler (Philox of
``sampler_seed``, epoch), the fused dropout masks (Philox of ``seed``, epoch), the flag sequence numbers
(``seq_base + epoch_dev``) -- so the state is small: the weights and buffers, Adam's moments and step, the seed, the
epochs completed, the evaluator's best model, and per rank torch's CUDA generator (``nn.Dropout`` of the op-by-op path
draws from it).  A resumed run computes what the uninterrupted run computes, bit for bit (DESIGN.md).

Layout, one filesystem shared by all ranks (as for the partition store)::

    checkpoint/<graph_name>_state/CURRENT              the name of the complete state, replaced atomically
    checkpoint/<graph_name>_state/epoch<N>-<id>/       shared.pt (rank 0) + rank<r>.pt (every rank)
    checkpoint/<graph_name>_state/incomplete/          the save in progress

A save writes into ``incomplete/``; after a barrier rank 0 renames it to a fresh ``epoch<N>-<id>`` and then points
``CURRENT`` at it (``os.replace``); only then is the previous state deleted.  A crash at any point leaves ``CURRENT``
naming a complete state, or no ``CURRENT`` at all before the first save completed.
"""
from __future__ import annotations

import copy
import os
import shutil
import uuid
from typing import Dict, List, Optional

import torch

from .helper import context as ctx

FORMAT = 1
_TMP, _CURRENT = "incomplete", "CURRENT"

# The arguments that decide the training trajectory, with the value a missing one stands for.  A state only resumes a
# run that agrees on all of them; --n-epochs, --log-every, the evaluation flags and the seed may differ (the seed is
# taken from the state).
FINGERPRINT = (
    ("model", None), ("n_layers", None), ("n_hidden", None), ("n_feat", None), ("n_class", None), ("heads", 1),
    ("norm", "layer"), ("n_linear", 0), ("use_pp", False), ("dropout", None), ("lr", None), ("weight_decay", 0.0),
    ("sampling_rate", None), ("sampler_seed", 0), ("n_partitions", None), ("graph_name", ""), ("backend", "nccl"),
    ("agg_dtype", "f32"), ("comm_dtype", "f32"), ("dense_dtype", "f32"),
)


def fingerprint(args: dict) -> dict:
    """The trajectory-deciding subset of an argument dict (``vars(args)``)."""
    return {k: args.get(k, default) for k, default in FINGERPRINT}


def fingerprint_mismatches(saved: dict, current: dict) -> List[str]:
    """One line per field of ``FINGERPRINT`` on which two argument dicts differ (empty: a state saved under ``saved``
    may resume a run with ``current``)."""
    a, b = fingerprint(saved), fingerprint(current)
    return [f"{k} is {b[k]!r}, the state's {a[k]!r}" for k, _ in FINGERPRINT if a[k] != b[k]]


def state_dir(args) -> str:
    """Beside the reference-format checkpoints (``evaluate.checkpoint_path``)."""
    return os.path.join('checkpoint', args.graph_name + '_state')


def _cpu(x):
    """A deep copy with every tensor on the host."""
    if isinstance(x, torch.Tensor):
        return x.detach().to('cpu', copy=True)
    if isinstance(x, dict):
        return {k: _cpu(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_cpu(v) for v in x)
    return x


def _write(path: str, obj) -> None:
    with open(path, 'wb') as f:
        torch.save(obj, f)
        f.flush()
        os.fsync(f.fileno())


def _sync_dir(path: str) -> None:
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def _path_kind(st) -> str:
    return "fused" if st.arena is not None else "op-by-op"


def save(st, epochs: int, evaluator=None) -> str:
    """Write the state after ``epochs`` completed epochs (collective: every rank calls it at the same epoch).  Returns
    the directory of the new state, current on every rank when this returns."""
    c = ctx.comm()
    root = state_dir(st.args)
    tmp = os.path.join(root, _TMP)
    if c.rank == 0:
        shutil.rmtree(tmp, ignore_errors=True)            # a save that crashed: never current, nothing to keep
        os.makedirs(tmp)
    c.barrier()
    dev = st.feat.device
    _write(os.path.join(tmp, f"rank{c.rank}.pt"), {"rank": c.rank, "cuda_rng": torch.cuda.get_rng_state(dev)})
    if c.rank == 0:
        best = getattr(evaluator, 'best_model', None)
        _write(os.path.join(tmp, "shared.pt"), {
            "format": FORMAT, "epochs": int(epochs), "seed": int(st.args.seed), "path": _path_kind(st),
            "fingerprint": fingerprint(vars(st.args)),
            "model": _cpu(st.model.state_dict()), "optimizer": _cpu(st.optimizer.state_dict()),
            "best_acc": getattr(evaluator, 'best_acc', None),
            "best_model": None if best is None else _cpu(best.state_dict())})
    c.barrier()                                           # every rank's file is on disk
    name = None
    if c.rank == 0:
        name = "epoch%08d-%s" % (epochs, uuid.uuid4().hex[:12])
        os.rename(tmp, os.path.join(root, name))
        _sync_dir(root)
        cur_tmp = os.path.join(root, _CURRENT + ".tmp")
        with open(cur_tmp, 'w') as f:
            f.write(name + "\n")
            f.flush()
            os.fsync(f.fileno())
        os.replace(cur_tmp, os.path.join(root, _CURRENT))
        _sync_dir(root)
        for d in os.listdir(root):                        # the previous state, now superseded
            if d.startswith("epoch") and d != name:
                shutil.rmtree(os.path.join(root, d), ignore_errors=True)
    c.barrier()
    return os.path.join(root, name) if name is not None else _current(root)


def _current(root: str) -> Optional[str]:
    try:
        with open(os.path.join(root, _CURRENT)) as f:
            name = f.read().strip()
    except FileNotFoundError:
        return None
    return os.path.join(root, name)


def load(args, rank: int) -> Dict:
    """This rank's view of the current state under ``args.graph_name``: the shared part plus its own.  Raises
    ``ValueError`` when there is no complete state, or when it was saved by a run with other trajectory-deciding
    arguments (naming every difference)."""
    root = state_dir(args)
    d = _current(root)
    if d is None or not os.path.isdir(d):
        tmp = os.path.join(root, _TMP)
        extra = f" (only an incomplete save in {tmp})" if os.path.isdir(tmp) else ""
        raise ValueError(f"--resume: no complete training state in {root}{extra}; run with --save-state-every first")
    shared = torch.load(os.path.join(d, "shared.pt"), map_location='cpu')
    why = fingerprint_mismatches(shared["fingerprint"], vars(args))
    if shared.get("format") != FORMAT:
        why.append(f"state format {shared.get('format')!r}, this build reads {FORMAT}")
    if why:
        raise ValueError(f"--resume: the state in {d} was saved by a different run: " + "; ".join(why))
    own = torch.load(os.path.join(d, f"rank{rank}.pt"), map_location='cpu')
    return dict(shared, dir=d, cuda_rng=own["cuda_rng"])


def restore(st, saved: Dict, evaluator=None) -> int:
    """Put a loaded state into a fresh ``train.setup`` result (and the run's evaluator); returns the epochs completed,
    the index of the next epoch.  The seed is set too, so a launch that drew a new one continues with the saved one."""
    if saved["path"] != _path_kind(st):
        raise ValueError(f"--resume: the state in {saved['dir']} was saved by the {saved['path']} training step, this "
                         f"run takes the {_path_kind(st)} one (BNS_FUSED); a state does not carry across")
    dev = st.feat.device
    st.args.seed = saved["seed"]
    st.model.load_state_dict(saved["model"])
    st.optimizer.load_state_dict(saved["optimizer"])
    if st.arena is not None:
        st.arena.refresh(advance=None)                    # W^T and bias sums of the loaded weights
    st.epoch_dev.fill_(saved["epochs"])                   # in place: the sampler / flags / masks read this counter
    torch.cuda.set_rng_state(saved["cuda_rng"], dev)
    if evaluator is not None and saved["best_model"] is not None:
        best = copy.deepcopy(st.model)                    # what Evaluator.after_epoch would have snapshotted
        best.load_state_dict(saved["best_model"])
        evaluator.best_acc, evaluator.best_model = saved["best_acc"], best
    return int(saved["epochs"])
