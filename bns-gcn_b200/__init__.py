"""bns-gcn_b200: the H100-native hot path of BNS-GCN (partition-parallel GCN training with
random boundary-node sampling) behind the reference's own Python surface.

Layout (mirrors the reference's tree so call sites read the same):
  csrc/      sm_90a CUDA kernels + the C-ABI (``include/bnsgcn.h``) -> ``libbnsgcn.so``
  _lib.py    ctypes binding of that library (fails loudly when it is missing)
  ops.py     ``torch.autograd.Function`` wrappers over the C-ABI calls
  module/    ``layer.py`` ``model.py``      (reference: module/layer.py, module/model.py)
  helper/    ``feature_buffer.py`` ``reducer.py`` ``utils.py`` ``parser.py`` ``context.py`` ``timer/``
  train.py   the epoch loop and its setup  (reference: train.py)
  data/      synthetic graphs + the partition contract (stand-in for DGL/OGB loaders)
"""
__version__ = "0.1.0"
