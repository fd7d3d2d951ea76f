"""``Buffer``: the sampled boundary-feature exchange (reference: helper/feature_buffer.py).

Same surface -- ``init_buffer(num_in, ratio, f_send_shape, f_recv_shape, layer_size, use_pp, backend)``,
``set_selected(selected)``, ``update(layer, feat) -> [n_U, F]`` whose gradient does the reverse exchange and the
``/ratio`` scatter-add (``__grad_hook``, :169-174) -- but nothing leaves the device:

* ``backend='nccl'`` (staged): pack kernel (K3, ``bns_gather_div_f32``) -> one grouped NCCL send/recv on a side
  stream straight into the tail rows of the concat buffer -> scatter-add kernel (K5) in backward.  Replaces the
  pinned-host gloo ring of :101-129.
* ``backend='p2p'``: the pack kernel of the sender stores ``H[selected]/ratio`` directly into the receiver's concat
  buffer through a peer-mapped pointer (NVLink 5 / NVSwitch) and raises a flag there (``bns_p2p_put_rows_f32`` /
  ``bns_p2p_wait_flag``): K3 + C1 fused, no staging copy, no NCCL launch.

``comm_dtype='bf16'`` (``--comm-dtype bf16``, fused GraphSAGE / GCN step only): the sender rounds each boundary row
``H[selected]/ratio`` -- and each returned gradient row -- to bf16 once, so the wire and the receiving slab carry half
the bytes.  ``update`` then returns the inner rows ``[n_in, F]`` (f32, as given) with the received halo rows attached
as ``_bns_halo`` (bf16 ``[recv_total, F]``), and the halo gradient travels only through ``begin_backward``.
``comm_dtype='fp8'`` (``--comm-dtype fp8``) does the same with fp8 rows (``ops.Fp8Rows``: e4m3 codes plus a power-of-two
scale per row, ``ops.cvt_rows_fp8``'s rule over the f32 quotients): ``F + 4`` bytes a row, and ``_bns_halo`` is an
``Fp8Rows`` view of the received codes and scales -- the gather table of the wide layers' halo pass as it arrived.

The exchange runs on ``self._comm_stream``; with ``update(..., overlap=True)`` the caller's stream does not wait
for it -- the aggregation op waits on ``h_u._bns_ready`` right before it touches the halo rows, so the transfer
hides behind the inner-edge SpMM.  ``Comm(s)`` is measured with CUDA events on that stream.
"""
from __future__ import annotations

import ctypes
import struct
from typing import List, Optional

import torch

from .. import ops
from .._lib import MAX_PEERS, P2P_HANDLE_BYTES, EpochMaps, PutAll, check, lib
from . import context as ctx
from .timer.timer import comm_timer


class _DevArray:
    """Zero-copy torch view of library-owned device memory (``__cuda_array_interface__``)."""

    def __init__(self, ptr: int, shape, typestr="<f4"):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False),
                                         "version": 2, "strides": None}


def _a256(n: int) -> int:
    return (n + 255) // 256 * 256


def slab_layout(n_in, recv_total, send_total, width, n_comm_layers, comm_dtype='f32') -> dict:
    """Byte layout of one rank's peer-mapped slab.  Per communicating layer: a forward region -- the ``n_in`` inner f32
    rows, then the ``recv_total`` received halo rows -- and a backward region of the ``send_total`` gradient rows this
    rank gets back; the received id lists close the slab.  With bf16 the halo and backward rows are bf16 and every
    sub-region starts on 256 bytes.  With fp8 the halo and backward rows are e4m3 codes, each followed by its region of
    f32 scales (``halo_scale_off`` / ``bwd_scale_off``), every sub-region on 256 bytes.  ``*_bytes``: the size of each
    region (one layer)."""
    if comm_dtype == 'fp8':
        n_h, n_b = max(recv_total, 1), max(send_total, 1)
        inner, halo, halo_s = _a256(n_in * width * 4), _a256(n_h * width), _a256(n_h * 4)
        bwd, bwd_s = _a256(n_b * width), _a256(n_b * 4)
        stride = inner + halo + halo_s + bwd + bwd_s
        fwd_off = [l * stride for l in range(n_comm_layers)]
        halo_off = [o + inner for o in fwd_off]
        halo_scale_off = [o + halo for o in halo_off]
        bwd_off = [o + halo_s for o in halo_scale_off]
        bwd_scale_off = [o + bwd for o in bwd_off]
        ids_off = n_comm_layers * stride
        return {"fwd_off": fwd_off, "halo_off": halo_off, "halo_scale_off": halo_scale_off, "bwd_off": bwd_off,
                "bwd_scale_off": bwd_scale_off, "ids_off": ids_off, "slab_bytes": ids_off + max(recv_total, 1) * 8,
                "inner_bytes": inner, "halo_bytes": halo, "halo_scale_bytes": halo_s, "bwd_bytes": bwd,
                "bwd_scale_bytes": bwd_s}
    if comm_dtype == 'bf16':
        inner, halo, bwd = _a256(n_in * width * 4), _a256(max(recv_total, 1) * width * 2), _a256(max(send_total, 1) * width * 2)
        stride = inner + halo + bwd
        fwd_off = [l * stride for l in range(n_comm_layers)]
        halo_off = [o + inner for o in fwd_off]
        bwd_off = [o + halo for o in halo_off]
        ids_off = n_comm_layers * stride
    else:
        row = width * 4
        inner, halo, bwd = n_in * row, recv_total * row, max(send_total, 1) * row
        fwd_off = [l * (inner + halo + bwd) for l in range(n_comm_layers)]
        halo_off = [o + inner for o in fwd_off]
        bwd_off = [o + inner + halo for o in fwd_off]
        ids_off = _a256(n_comm_layers * (inner + halo + bwd))
    return {"fwd_off": fwd_off, "halo_off": halo_off, "bwd_off": bwd_off, "ids_off": ids_off,
            "slab_bytes": ids_off + max(recv_total, 1) * 8, "inner_bytes": inner, "halo_bytes": halo, "bwd_bytes": bwd}


def wire_bytes(send_total, recv_total, F, comm_dtype='f32') -> dict:
    """Feature bytes one rank moves per communicating layer and epoch: forward it sends its ``send_total`` sampled rows
    and receives ``recv_total`` halo rows; backward the reverse.  An fp8 row is ``F`` codes and one f32 scale."""
    row = F + 4 if comm_dtype == 'fp8' else F * (2 if comm_dtype == 'bf16' else 4)
    return {"fwd_send": send_total * row, "fwd_recv": recv_total * row,
            "bwd_send": recv_total * row, "bwd_recv": send_total * row}


class Buffer(object):

    def __init__(self):
        super(Buffer, self).__init__()
        self._num_in = None
        self._selected: List[Optional[torch.Tensor]] = []
        self._n_layers = 0
        self._layer_size = []
        self._ratio = []
        self._recv_shape, self._send_shape = [], []
        self._backend = None
        self._pl, self._pr = [], []
        self._comm_stream = None
        self._send_buf, self._b_recv = None, None
        self._p2p = None
        self._seq = {}
        # CUDA-graph mode (train.GraphedEpoch): no timing events; flag sequence numbers = seq_base + *seq_dev
        self.graph_mode = False
        self.stamps = None                      # a timed capture: timer.ReplayStamps in place of the events
        self.seq_dev = None
        self.seq_base = 0
        self._maps = None
        self._comm_dtype = 'f32'
        self._bf16 = self._fp8 = False
        self._apart = False                     # bf16 / fp8: the halo rows travel and are returned apart from feat

    # helper/feature_buffer.py:23-33
    def __init_pl_pr(self):
        self._pl, self._pr = [], []
        tot = self._num_in
        for j, s in enumerate(self._recv_shape):
            if j == self._rank:
                self._pl.append(None)
                self._pr.append(None)
            else:
                self._pl.append(tot)
                tot += s
                self._pr.append(tot)
        self._n_u = tot

    def init_buffer(self, num_in, ratio, f_send_shape, f_recv_shape, layer_size, use_pp=False, backend='nccl',
                    device=None, comm_dtype='f32'):
        if use_pp is False:
            raise NotImplementedError            # helper/feature_buffer.py:36-37
        if comm_dtype not in ('f32', 'bf16', 'fp8'):
            raise ValueError(f"comm_dtype {comm_dtype!r}: expected 'f32', 'bf16' or 'fp8'")
        c = ctx.comm()
        # captured now: backward runs on autograd's device thread, where thread-local lookups would miss
        self._comm, self._timer = c, comm_timer._get()
        self._rank, self._size = c.rank, c.size
        self._num_in = num_in
        self._n_layers = len(layer_size)
        self._layer_size = layer_size
        self._recv_shape = [int(s) for s in f_recv_shape]
        self._send_shape = [int(s) for s in f_send_shape]
        self._ratio = ratio
        if backend in ('nccl', 'staged'):
            backend = 'nccl'
        elif backend != 'p2p':
            raise NotImplementedError(f"backend {backend!r}: this build moves boundary rows GPU-to-GPU "
                                      "('nccl' or 'p2p'); the reference's host-staged gloo/mpi paths are what it replaces")
        self._backend = backend
        self.__init_pl_pr()
        if self._size == 1:
            return
        self._device = torch.device(device if device is not None else torch.cuda.current_device())
        if self._device.type != 'cuda':
            raise RuntimeError("Buffer needs a CUDA device: there is no CPU exchange path")
        width = self._layer_size[1]              # the reference sizes every slab with layer_size[1] (:54-55)
        self._width = width
        self._comm_dtype = comm_dtype
        self._bf16, self._fp8 = comm_dtype == 'bf16', comm_dtype == 'fp8'
        self._apart = self._bf16 or self._fp8
        if self._bf16 and width % 8:
            raise ValueError(f"comm_dtype bf16: exchanged width {width} is not a multiple of 8")
        if self._fp8 and width % 16:
            raise ValueError(f"comm_dtype fp8: exchanged width {width} is not a multiple of 16")
        wire = torch.bfloat16 if self._bf16 else torch.float32
        self._comm_stream = torch.cuda.Stream(self._device)
        self._send_begin, tot = [], 0
        for j in range(self._size):
            self._send_begin.append(tot)
            tot += 0 if j == self._rank else self._send_shape[j]
        self._send_total = tot
        if backend == 'nccl':
            def rows(n):
                return self._fp8_rows(n) if self._fp8 else torch.zeros(n, width, dtype=wire, device=self._device)
            self._send_buf = [None if j == self._rank else rows(self._send_shape[j]) for j in range(self._size)]
            self._b_recv = [None if j == self._rank else rows(self._send_shape[j]) for j in range(self._size)]
            # bf16 / fp8: the halo gradient rows are rounded into this buffer before they are sent (f32 sends them in
            # place)
            self._b_send = rows(max(self._n_u - num_in, 1)) if self._apart else None
        else:
            self.__init_p2p(c, width)

    # ---- p2p slabs -------------------------------------------------------------------------------
    def __init_p2p(self, c, width):
        n_comm_layers = max(self._n_layers - 1, 1)
        if self._size - 1 > MAX_PEERS:
            raise RuntimeError(f"p2p transport: at most {MAX_PEERS + 1} partitions (BNS_MAX_PEERS)")
        self._hop_begin, tot = [], 0
        for j in range(self._size):
            self._hop_begin.append(tot)
            tot += 0 if j == self._rank else self._recv_shape[j]
        self._recv_total = tot
        # after the feature regions: the received id lists of the epoch (data_transfer NODE), int64 [sum of recv sizes]
        lay = slab_layout(self._num_in, tot, self._send_total, width, n_comm_layers, self._comm_dtype)
        self._fwd_off, self._halo_off, self._bwd_off, self._ids_off = (lay["fwd_off"], lay["halo_off"], lay["bwd_off"],
                                                                       lay["ids_off"])
        self._halo_scale_off, self._bwd_scale_off = lay.get("halo_scale_off"), lay.get("bwd_scale_off")
        slab_bytes = lay["slab_bytes"]
        self._n_comm_layers = n_comm_layers
        n_flags = (n_comm_layers * 2 + 1) * self._size          # (layer, direction, source) + (ids, source)
        # completion tickets of the all-peer puts: size + 2 (layer - 1) forward, + 1 backward, size + 2 n_comm_layers
        # the ids -- all below size + n_flags, which the library provides for any depth
        h = ctypes.c_void_p()
        with torch.cuda.device(self._device):
            check(lib.bns_p2p_create(ctypes.byref(h), self._rank, self._size, slab_bytes, n_flags), "bns_p2p_create")
        self._p2p = h
        slab, flags, nbytes = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_size_t()
        check(lib.bns_p2p_local(h, ctypes.byref(slab), ctypes.byref(flags), ctypes.byref(nbytes)), "bns_p2p_local")
        self._slab_ptr = slab.value
        # publish: where peers must write inside MY slab (row offsets of their segment) + how to map my memory
        my = {"fwd_off": self._fwd_off, "halo_off": self._halo_off, "bwd_off": self._bwd_off, "pl": self._pl,
              "send_begin": self._send_begin, "halo_scale_off": self._halo_scale_off, "bwd_scale_off": self._bwd_scale_off,
              "ids_off": self._ids_off, "hop_begin": self._hop_begin, "slab_bytes": nbytes.value}
        if c.kind == "thread":
            my["ptrs"] = (slab.value, flags.value)
        else:
            hb = ctypes.create_string_buffer(2 * P2P_HANDLE_BYTES)
            check(lib.bns_p2p_export(h, hb), "bns_p2p_export")
            my["handle"] = hb.raw
        import pickle
        table = [pickle.loads(b) for b in c.all_gather_bytes(pickle.dumps(my))]
        self._peer_layout = table
        for j in range(self._size):
            if j == self._rank:
                continue
            if c.kind == "thread":
                check(lib.bns_p2p_set_peer(h, j, table[j]["ptrs"][0], table[j]["ptrs"][1], table[j]["slab_bytes"]),
                      "bns_p2p_set_peer")
            else:
                with torch.cuda.device(self._device):
                    check(lib.bns_p2p_import(h, j, table[j]["handle"], table[j]["slab_bytes"]), "bns_p2p_import")
        c.barrier()
        self._peers = [j for j in range(self._size) if j != self._rank]               # ascending: segment order
        self._ring_out = [(self._rank + i) % self._size for i in range(1, self._size)]
        self._ring_in = [(self._rank - i + self._size) % self._size for i in range(1, self._size)]

    # ---- per-epoch ids and maps (p2p transport) ------------------------------------------------------
    def set_maps(self, maps: torch.Tensor, n_halo: int, pos):
        """``maps``: ONE int32 allocation ``[n_halo + (P-1) * n_in]`` = the slot map of the partition graph followed by
        the inverse map of every peer (ascending); ``pos``: train.get_pos()."""
        self._maps, self._n_halo, self._pos = maps, n_halo, pos
        self._inv = {}
        for s_, j in enumerate(self._peers):
            b = n_halo + s_ * self._num_in
            self._inv[j] = maps[b:b + self._num_in]

    def uses_p2p_ids(self) -> bool:
        return self._p2p is not None and self._maps is not None

    def exchange_ids(self, sel_cat: torch.Tensor):
        """data_transfer(selected, ..., tag=NODE) (helper/utils.py:187-213, train.py:389) over peer memory: one kernel
        stores every peer's sampled id list into that peer's slab and raises its flag, one kernel waits for the lists of
        all peers.  Returns ``(one_hops_cat, [per-peer views])`` -- views of this rank's slab."""
        cs = self._comm_stream
        main = torch.cuda.current_stream(self._device)
        n = len(self._peers)
        begin = (ctypes.c_int64 * (n + 1))()
        peers = (ctypes.c_int32 * max(n, 1))()
        roff = (ctypes.c_uint64 * max(n, 1))()
        tot = 0
        for s_, j in enumerate(self._peers):
            begin[s_] = tot
            tot += self._send_shape[j]
            peers[s_] = j
            lay = self._peer_layout[j]
            roff[s_] = lay["ids_off"] + lay["hop_begin"][self._rank] * 8
        begin[n] = tot
        flag_base = self._n_comm_layers * 2 * self._size
        seq, seq_dev = self._seq_args("ids", False)
        start = torch.cuda.Event()
        start.record(main)
        cs.wait_event(start)
        with torch.cuda.stream(cs):
            check(lib.bns_p2p_put_ids_i64(self._p2p, n, begin, peers, roff, sel_cat.data_ptr() if tot else None,
                                          flag_base + self._rank, self._size + 2 * self._n_comm_layers, seq, seq_dev,
                                          cs.cuda_stream),
                  "bns_p2p_put_ids_i64")
            for j in self._peers:
                self._post_put_event(j, 1999, cs)
            for j in self._peers:
                self._await_put_event(j, 1999, cs)
            idx = (ctypes.c_int32 * max(n, 1))(*[flag_base + j for j in self._peers])
            check(lib.bns_p2p_wait_all(self._p2p, n, idx, seq, seq_dev, cs.cuda_stream), "bns_p2p_wait_all")
            done = torch.cuda.Event()
            done.record(cs)
        if not self.graph_mode:
            sel_cat.record_stream(cs)
        main.wait_event(done)
        # a private copy: the slab region is rewritten by the peers at the start of THEIR next epoch, and the lists stay
        # visible to the caller (train.TrainState.one_hops) after this epoch has ended
        cat = torch.as_tensor(_DevArray(self._slab_ptr + self._ids_off, (max(self._recv_total, 1),), "<i8"),
                              device=self._device)[:self._recv_total].clone()
        views = [None] * self._size
        for j in self._peers:
            views[j] = cat[self._hop_begin[j]:self._hop_begin[j] + self._recv_shape[j]]
        return cat, views

    def update_maps(self, sel_cat: torch.Tensor, hops_cat: torch.Tensor, slot: torch.Tensor):
        """construct_graph (train.py:256-281) for all peers + the inverse maps of the gradient scatter: one memset, one
        kernel (``bns_epoch_maps_update``)."""
        m = EpochMaps()
        n = len(self._peers)
        m.n_seg = n
        a = b = 0
        for s_, j in enumerate(self._peers):
            m.sel_begin[s_], m.hop_begin[s_] = a, b
            a += self._send_shape[j]
            b += self._recv_shape[j]
            m.pos[s_] = self._pos[j].data_ptr()
            m.inv[s_] = self._inv[j].data_ptr()
        m.sel_begin[n], m.hop_begin[n] = a, b
        m.selected_cat = sel_cat.data_ptr() if a else None
        m.one_hops_cat = hops_cat.data_ptr() if b else None
        m.slot = slot.data_ptr()
        m.n_in = self._num_in
        with torch.cuda.device(self._device):
            check(lib.bns_epoch_maps_update(ctypes.byref(m), self._maps.data_ptr(), self._maps.numel() * 4,
                                            torch.cuda.current_stream(self._device).cuda_stream), "bns_epoch_maps_update")

    # Ranks that are THREADS of one process share a CUDA context, where a kernel spinning on a flag can block the
    # very launch that would set it (lazy module loading and stream->hardware-queue aliasing both synchronise the
    # context).  There, the producer hands over an event recorded after its put and the consumer's stream waits on
    # it BEFORE the flag-wait kernel is launched, so that kernel finds the flag already set and never spins.  With
    # one process per GPU (the deployment shape) these two calls do nothing and the flag is the only signal.
    def _post_put_event(self, peer, tag, stream):
        if self._comm.kind == "thread":
            ev = torch.cuda.Event()
            ev.record(stream)
            self._comm.post_event(peer, tag, ev)

    def _await_put_event(self, peer, tag, stream):
        if self._comm.kind == "thread":
            stream.wait_event(self._comm.take_event(peer, tag))

    def _timer_ctx(self, name, stream):
        import contextlib
        if not self.graph_mode:
            return self._timer.timer(name, stream=stream)
        return self.stamps.interval(name, stream) if self.stamps is not None else contextlib.nullcontext()

    def _seq_args(self, layer, backward):
        """(immediate, device pointer) of this exchange's flag value."""
        if self.graph_mode:
            return self.seq_base, self.seq_dev.data_ptr()
        key = (layer, 1 if backward else 0)
        self._seq[key] = self._seq.get(key, 0) + 1
        return self._seq[key], None

    def _esz(self):
        """Bytes per element of a row on the wire (an fp8 row's scale lives apart)."""
        return 1 if self._fp8 else 2 if self._bf16 else 4

    def _flag(self, layer, backward, src):
        return ((layer - 1) * 2 + (1 if backward else 0)) * self._size + src

    def _fp8_rows(self, rows, alloc=torch.zeros):
        """An ``ops.Fp8Rows`` of ``rows`` rows of the slab width (the staged transport's buffers)."""
        return ops.Fp8Rows(alloc(rows, self._width, dtype=torch.float8_e4m3fn, device=self._device),
                           alloc(rows, dtype=torch.float32, device=self._device))

    def _slab_fp8(self, codes_off, scale_off, rows):
        """``ops.Fp8Rows`` view of ``rows`` code rows of the slab width and their scales in this rank's slab."""
        codes = torch.as_tensor(_DevArray(self._slab_ptr + codes_off, (rows, self._width), "|u1"), device=self._device)
        scale = torch.as_tensor(_DevArray(self._slab_ptr + scale_off, (rows,)), device=self._device)
        return ops.Fp8Rows(codes.view(torch.float8_e4m3fn), scale)

    def _alltoall(self, send, recv, tag):
        """``comm.alltoall``; fp8 rows go as two messages per peer, their codes (as bytes), then their scales."""
        if not self._fp8:
            return self._comm.alltoall(send, recv, tag=tag)
        for part in (lambda r: r.codes.view(torch.uint8), lambda r: r.scale):
            self._comm.alltoall([None if r is None else part(r) for r in send],
                                [None if r is None else part(r) for r in recv], tag=tag)

    def _slab_view(self, byte_off, rows, bf16=False):
        if bf16:
            return torch.as_tensor(_DevArray(self._slab_ptr + byte_off, (rows, self._width), "<i2"),
                                   device=self._device).view(torch.bfloat16)
        return torch.as_tensor(_DevArray(self._slab_ptr + byte_off, (rows, self._width)), device=self._device)

    def input_slot(self, layer, rows, width):
        """The rows ``[0, n_in)`` of layer ``layer``'s concat buffer when they can be written in place (peer-mapped
        transport, full slab width), else None.  ``update(layer, feat)`` recognises a ``feat`` that already lives there
        and skips its copy (K4)."""
        if self._size == 1 or self._p2p is None or rows != self._num_in or width != getattr(self, "_width", -1):
            return None
        if not (1 <= layer <= self._n_comm_layers):
            return None
        return self._slab_view(self._fwd_off[layer - 1], self._num_in)

    def set_selected(self, selected, selected_cat=None):
        """``selected_cat``: the same lists concatenated in ascending peer order (what the sampler produced); built here
        when the caller injects per-peer lists."""
        self._selected = selected
        if selected_cat is None and self._p2p is not None:
            parts = [selected[j] for j in self._peers if selected[j] is not None and selected[j].numel()]
            selected_cat = torch.cat(parts) if parts else torch.empty(0, dtype=torch.int64, device=self._device)
        self._selected_cat = selected_cat

    # ---- forward ---------------------------------------------------------------------------------
    def update(self, layer, feat, overlap=False):
        """``[feat ; recv_0 ; recv_1 ...]`` with the boundary rows of the peers (helper/feature_buffer.py:93-99)."""
        if self._size == 1:
            return feat
        res = _BoundaryExchange.apply(feat, self, layer, overlap)
        if overlap:
            res._bns_ready = self._last_ready
        res._bns_exchange = (self, layer)          # lets a fused consumer start the gradient return trip early
        if self._apart:
            res._bns_halo = self._last_halo        # the received rows, bf16 / fp8: the layer gathers / widens them itself
        return res

    def _forward(self, layer, feat, overlap):
        F = feat.shape[1]
        if F > self._width:
            raise RuntimeError(f"layer width {F} > slab width {self._width} (the reference sizes slabs with layer_size[1])")
        feat = feat.contiguous()
        main, cs = torch.cuda.current_stream(self._device), self._comm_stream
        ready = torch.cuda.Event()
        bf16, fp8, apart, halo = self._bf16, self._fp8, self._apart, None
        if (self._p2p is not None or fp8) and F != self._width:
            raise RuntimeError(f"{'p2p transport' if self._p2p is not None else 'comm_dtype fp8'} needs equal hidden "
                               "widths")
        if apart:
            # the inner rows go on as they are (no concat); the halo rows land in a bf16 / fp8 table of their own
            h_u, n_halo = feat, self._n_u - self._num_in
            if self._backend == 'nccl':
                halo = (self._fp8_rows(n_halo, torch.empty) if fp8 else
                        torch.empty(n_halo, F, dtype=torch.bfloat16, device=self._device))
            elif fp8:
                halo = self._slab_fp8(self._halo_off[layer - 1], self._halo_scale_off[layer - 1], max(n_halo, 1))[:n_halo]
            else:
                halo = self._slab_view(self._halo_off[layer - 1], max(n_halo, 1), bf16=True)[:n_halo]
        elif self._backend == 'nccl':
            h_u = torch.empty(self._n_u, F, device=self._device)
        else:
            h_u = self._slab_view(self._fwd_off[layer - 1], self._n_u)[:, :F]
        if feat.data_ptr() != h_u.data_ptr():                          # (written in place by the producer: input_slot)
            ops.copy_rows(feat, h_u, self._num_in)                     # K4: the only copy of the concat
        start = torch.cuda.Event()
        start.record(main)
        cs.wait_event(start)
        with torch.cuda.stream(cs):
            with self._timer_ctx(f'forward_{layer}', cs):
                if self._backend == 'nccl':
                    send = [None] * self._size
                    recv = [None] * self._size
                    for j in range(self._size):
                        if j == self._rank:
                            continue
                        send[j] = self._send_buf[j] if fp8 else self._send_buf[j][:, :F] if F == self._width else \
                            torch.empty(self._send_shape[j], F, dtype=self._send_buf[j].dtype, device=self._device)
                        ops.gather_div(feat, self._selected[j], self._ratio[j], out=send[j])      # K3
                        recv[j] = (halo[self._pl[j] - self._num_in:self._pr[j] - self._num_in] if apart else
                                   h_u[self._pl[j]:self._pr[j]])
                    self._alltoall(send, recv, 16 + layer)                                        # C1/C2
                else:
                    seq, seq_dev = self._seq_args(layer, False)
                    segs = PutAll()
                    segs.n_seg = len(self._peers)
                    scale_off = (ctypes.c_uint64 * max(len(self._peers), 1))()
                    tot = 0
                    for s_, j in enumerate(self._peers):
                        lay = self._peer_layout[j]
                        segs.row_begin[s_] = tot
                        tot += self._send_shape[j]
                        segs.peer[s_] = j
                        if fp8:
                            segs.remote_off[s_] = lay["halo_off"][layer - 1] + lay["hop_begin"][self._rank] * self._width
                            scale_off[s_] = lay["halo_scale_off"][layer - 1] + lay["hop_begin"][self._rank] * 4
                        elif bf16:
                            segs.remote_off[s_] = lay["halo_off"][layer - 1] + lay["hop_begin"][self._rank] * self._width * 2
                        else:
                            segs.remote_off[s_] = lay["fwd_off"][layer - 1] + lay["pl"][self._rank] * self._width * 4
                        segs.div[s_] = float(self._ratio[j]) if self._send_shape[j] else 1.0
                    segs.row_begin[segs.n_seg] = tot
                    sel_cat = self._selected_cat
                    put = f"bns_p2p_put_all_{self._comm_dtype}"
                    check(getattr(lib, put)(self._p2p, ctypes.byref(segs), *((scale_off,) if fp8 else ()), self._width,
                                            feat.data_ptr(), feat.stride(0), F, sel_cat.data_ptr() if tot else None,
                                            self._flag(layer, False, self._rank), self._size + (layer - 1) * 2, seq,
                                            seq_dev, cs.cuda_stream), put)
                    for j in self._peers:
                        self._post_put_event(j, 2000 + 2 * layer, cs)
                    for j in self._peers:
                        self._await_put_event(j, 2000 + 2 * layer, cs)
                    idx = (ctypes.c_int32 * len(self._peers))(*[self._flag(layer, False, j) for j in self._peers])
                    check(lib.bns_p2p_wait_all(self._p2p, len(self._peers), idx, seq, seq_dev, cs.cuda_stream),
                          "bns_p2p_wait_all")
            ready.record(cs)
        if not self.graph_mode:
            feat.record_stream(cs)
            (halo.codes if fp8 else halo if bf16 else h_u).record_stream(cs)
            if fp8:
                halo.scale.record_stream(cs)
        if not overlap:
            main.wait_event(ready)
        self._last_ready, self._last_halo = ready, halo
        return h_u

    # ---- backward (the grad hook) -------------------------------------------------------------------
    def begin_backward(self, layer, grad):
        """Start the gradient return trip of ``layer`` as soon as the HALO rows ``grad[n_in:]`` are final: the rows go to
        their owners on the comm stream while the caller still computes ``grad[:n_in]`` (fused.SageConvFn.backward calls
        this between its two transposed aggregations).  ``_backward`` then only waits and scatter-adds."""
        if self._size == 1:
            return
        self._begun = (layer, grad.data_ptr(), self._exchange_backward(layer, grad))

    def _exchange_backward(self, layer, grad):
        """Enqueue send + receive of the halo gradient rows; returns ``(done event, recv list or None)``."""
        F = grad.shape[1]
        main, cs = torch.cuda.current_stream(self._device), self._comm_stream
        start, done = torch.cuda.Event(), torch.cuda.Event()
        start.record(main)
        cs.wait_event(start)
        recv = None
        with torch.cuda.stream(cs):
            with self._timer_ctx(f'backward_{layer}', cs):
                if self._backend == 'nccl':
                    # bf16 / fp8: the sender rounds its halo gradient rows once, then sends them per peer
                    rows = grad
                    if self._fp8:
                        halo = grad[self._num_in:]
                        rows = ops.cvt_rows_fp8(halo, out=self._b_send[:halo.shape[0]])
                    elif self._bf16:
                        halo = grad[self._num_in:]
                        rows = (ops.cvt_rows_bf16(halo, out=self._b_send[:halo.shape[0]]) if F == self._width else
                                ops.cvt_rows_bf16(halo))
                    b0 = self._num_in if self._apart else 0
                    send = [None if j == self._rank else rows[self._pl[j] - b0:self._pr[j] - b0] for j in range(self._size)]
                    recv = [None if j == self._rank else
                            (self._b_recv[j] if self._fp8 else self._b_recv[j][:, :F] if F == self._width else
                             torch.empty(self._send_shape[j], F, dtype=self._b_recv[j].dtype, device=self._device))
                            for j in range(self._size)]
                    self._alltoall(send, recv, 64 + layer)
                else:
                    seq, seq_dev = self._seq_args(layer, True)
                    segs = PutAll()
                    segs.n_seg = len(self._peers)
                    scale_off = (ctypes.c_uint64 * max(len(self._peers), 1))()
                    tot = 0
                    for s_, j in enumerate(self._peers):
                        lay = self._peer_layout[j]
                        segs.row_begin[s_] = tot
                        tot += self._recv_shape[j]
                        segs.peer[s_] = j
                        segs.remote_off[s_] = (lay["bwd_off"][layer - 1] +
                                               lay["send_begin"][self._rank] * self._width * self._esz())
                        if self._fp8:
                            scale_off[s_] = lay["bwd_scale_off"][layer - 1] + lay["send_begin"][self._rank] * 4
                        segs.src_begin[s_] = self._pl[j]
                        segs.div[s_] = 1.0
                    segs.row_begin[segs.n_seg] = tot
                    put = f"bns_p2p_put_all_{self._comm_dtype}"
                    check(getattr(lib, put)(self._p2p, ctypes.byref(segs), *((scale_off,) if self._fp8 else ()),
                                            self._width, grad.data_ptr(), grad.stride(0), F, None,
                                            self._flag(layer, True, self._rank), self._size + (layer - 1) * 2 + 1, seq,
                                            seq_dev, cs.cuda_stream), put)
                    for j in self._peers:
                        self._post_put_event(j, 2001 + 2 * layer, cs)
                    for j in self._peers:
                        self._await_put_event(j, 2001 + 2 * layer, cs)
                    idx = (ctypes.c_int32 * len(self._peers))(*[self._flag(layer, True, j) for j in self._peers])
                    check(lib.bns_p2p_wait_all(self._p2p, len(self._peers), idx, seq, seq_dev, cs.cuda_stream),
                          "bns_p2p_wait_all")
                    recv = [None] * self._size
                    n_b = max(self._send_total, 1)
                    bwd = (self._slab_fp8(self._bwd_off[layer - 1], self._bwd_scale_off[layer - 1], n_b) if self._fp8 else
                           self._slab_view(self._bwd_off[layer - 1], n_b, bf16=self._bf16)[:, :F])
                    for j in self._peers:
                        recv[j] = bwd[self._send_begin[j]:self._send_begin[j] + self._send_shape[j]]
            done.record(cs)
        if not self.graph_mode:
            grad.record_stream(cs)
        return done, recv

    def _backward(self, layer, grad):
        F = grad.shape[1]
        if not grad.is_contiguous():
            grad = grad.contiguous()
        trace = getattr(self, "trace", None)          # tests only: {name: tensor} of the gradients around the exchange
        if trace is not None:
            trace[f"grad_u{layer}"] = grad.detach().clone()
        main = torch.cuda.current_stream(self._device)
        begun, self._begun = getattr(self, "_begun", None), None
        if begun is not None and begun[0] == layer and begun[1] == grad.data_ptr():
            done, recv = begun[2]                     # the producer already sent the halo rows (begin_backward)
        elif self._apart:
            raise RuntimeError(f"comm_dtype {self._comm_dtype}: the layer that consumed the exchange must hand its halo "
                               "gradient to Buffer.begin_backward (the fused GraphSAGE / GCN layers do)")
        else:
            done, recv = self._exchange_backward(layer, grad)
        main.wait_event(done)
        inner = grad[:self._num_in]
        if self._backend == 'nccl' or self._maps is None:
            for i in range(1, self._size):           # the reference's order: idx = left, i = 1 .. P-1 (:111-129)
                left = (self._rank - i + self._size) % self._size
                ops.scatter_add_div(inner, self._selected[left], recv[left], self._ratio[left])      # K5
        else:
            # the same P-1 scatter-adds, in the same order, as ONE race-free launch over the inverse maps
            order = [j for j in self._ring_in if self._send_shape[j] > 0]
            if order:
                n = len(order)
                inv = (ctypes.c_void_p * n)(*[self._inv[j].data_ptr() for j in order])
                base = self._slab_ptr + self._bwd_off[layer - 1]
                rcv = (ctypes.c_void_p * n)(*[base + self._send_begin[j] * self._width * self._esz() for j in order])
                scl = ()
                if self._fp8:
                    sb = self._slab_ptr + self._bwd_scale_off[layer - 1]
                    scl = ((ctypes.c_void_p * n)(*[sb + self._send_begin[j] * 4 for j in order]),)
                div = (ctypes.c_float * n)(*[float(self._ratio[j]) for j in order])
                fn = f"bns_scatter_rows_all_{self._comm_dtype}"
                with torch.cuda.device(self._device):
                    check(getattr(lib, fn)(inner.data_ptr(), inner.stride(0), self._num_in, F, n, inv, rcv, *scl,
                                           self._width, div, main.cuda_stream), fn)
        if trace is not None:
            trace[f"grad_h{layer}"] = inner.detach().clone()
        return inner

    def __del__(self):
        h, self._p2p = getattr(self, "_p2p", None), None
        if h:
            try:
                lib.bns_p2p_destroy(h)
            except Exception:
                pass


class _BoundaryExchange(torch.autograd.Function):

    @staticmethod
    def forward(ctx_, feat, buf: Buffer, layer: int, overlap: bool):
        ctx_.buf, ctx_.layer = buf, layer
        return buf._forward(layer, feat, overlap)

    @staticmethod
    def backward(ctx_, grad):
        return ctx_.buf._backward(ctx_.layer, grad), None, None, None
