"""Halo-strip transports for the spatial layers.

Replaces the reference's tagged `dist.isend/irecv` on CUDA-aware MPI with a device-wide
`torch.cuda.synchronize()` before every message (spatial.py:336-403):

* PeerTransport (default on GPUs of one node): every rank owns one cudaMalloc'ed *mailbox*
  arena, mapped into its neighbours with CUDA IPC.  One pack kernel (spc_halo_pack) writes all
  outgoing strips straight into the neighbours' arenas over NVLink/NVSwitch (P2P stores), then a
  release-store at system scope publishes a per-slot sequence number; the receiver's stream
  waits on the flag with an acquire-load spin kernel.  No host synchronisation, no tags.
* DistTransport: the same strips through `torch.distributed.batch_isend_irecv` (NCCL on GPUs,
  gloo on CPU for the plumbing tests).  Selected with SPCONV_HALO_TRANSPORT=dist, or automatically --
  by a collective vote of all ranks at the first exchange -- when any rank cannot use peer mapping
  (ranks on more than one host, no CUDA IPC in the container).

`exchange_strips()` is the device-agnostic communication core (used by DistTransport and by the
CPU/gloo tests of the neighbour arithmetic).
"""
import ctypes as C
import os

import torch
import torch.distributed as dist

from .. import _lib

_DIRS = [(-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 0), (0, 1), (1, -1), (1, 0), (1, 1)]


def strip_shape(i, N, Cc, H, W, hh, hw):
    """Shape of strip i (reference spatial.py:311-334 get_shapes_recv)."""
    dr, dc = _DIRS[i]
    return (N, Cc, H if dr == 0 else hh, W if dc == 0 else hw)


def exchange_strips(send, recv, ranks, group=None):
    """Send send[i] to ranks[i] and receive recv[i] from ranks[i] for every i with a neighbour.
    Strip i travels to the neighbour in direction i, who receives it as ITS strip 8-i (the
    reference pairs send tag[i] with recv tag[8-i], spatial.py:170-172).  Between any ordered
    pair of ranks there is at most one strip per exchange, so no tags are needed."""
    ops = []
    for i in range(9):
        if i == 4 or send[i] is None:
            continue
        ops.append(dist.P2POp(dist.isend, send[i], ranks[i], group))
        ops.append(dist.P2POp(dist.irecv, recv[i], ranks[i], group))
    if not ops:
        return
    for req in dist.batch_isend_irecv(ops):
        req.wait()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _pack(x, hh, hw, ptrs):
    L = _lib.lib()
    N, Cc, H, W = x.shape
    arr = (C.c_void_p * 9)(*[C.c_void_p(p) if p else C.c_void_p(None) for p in ptrs])
    _lib.check(L.spc_halo_pack(N, Cc, H, W, hh, hw, _lib.dtype_code(x.dtype), C.c_void_p(x.data_ptr()),
                               C.byref(arr), _stream()), "spc_halo_pack")


class DistTransport:
    name = "dist"

    def exchange(self, layer, x, hh, hw, mask, ranks):
        N, Cc, H, W = x.shape
        send = [None] * 9
        recv = [None] * 9
        for i in range(9):
            if i != 4 and mask[i]:
                shp = strip_shape(i, N, Cc, H, W, hh, hw)
                send[i] = torch.empty(shp, dtype=x.dtype, device=x.device)
                recv[i] = torch.empty(shp, dtype=x.dtype, device=x.device)
        _pack(x, hh, hw, [t.data_ptr() if t is not None else 0 for t in send])
        exchange_strips(send, recv, ranks)
        return recv

    def reverse(self, layer, grads, shape, hh, hw, mask, ranks):
        """Reverse exchange of the exact backward: send the fp32 strip gradients grads[d] to neighbour d and return
        the ones the neighbours send back (recv[e] belongs to this tile's edge band e).  Same pairing as exchange()."""
        N, Cc, H, W = shape
        recv = [None] * 9
        for i in range(9):
            if i != 4 and mask[i]:
                recv[i] = torch.empty(strip_shape(i, N, Cc, H, W, hh, hw), dtype=torch.float32, device=grads[i].device)
        exchange_strips(grads, recv, ranks)
        return recv


class _CudaMem:
    """Expose raw device memory to torch through __cuda_array_interface__."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


class PeerTransport:
    """CUDA-IPC mailbox transport (see module docstring).  Every (layer, input shape) owns a slot
    in this rank's arena: two halves (double buffering by the parity of the exchange's sequence
    number) of packed receive areas, plus a block of flag words.  Slots are placed by a local bump
    allocator in first-use order, which may differ between ranks (a process that hosts the spatial
    layers of two models, GEMS-master + SP, visits them in a rank-dependent order): a sender
    therefore never assumes its neighbour's offsets -- the two ranks swap (data offset, flag base,
    slot bytes) once per (layer, neighbour) through torch.distributed at the first exchange."""

    name = "peer"
    # arrival[2][9] + ack[2][9] + post counter + collect counter + sequence word (+1 spare)
    FLAGS_PER_LAYER = 40
    _CNT_POST, _CNT_COLLECT, _SEQ = 36, 37, 38

    def __init__(self, device):
        self.device = device
        L = _lib.lib()
        self.arena_bytes = int(os.environ.get("SPCONV_ARENA_MB", "256")) << 20
        self.nflags = 1 << 16
        mb = C.c_void_p()
        _lib.check(L.spc_mailbox_create(C.byref(mb), self.arena_bytes, self.nflags), "spc_mailbox_create")
        self.mb = mb
        self.base = L.spc_mailbox_data(mb)
        self.arena = torch.as_tensor(_CudaMem(self.base, self.arena_bytes), device=device)
        handle = C.create_string_buffer(_lib.IPC_HANDLE_BYTES)
        _lib.check(L.spc_mailbox_export(mb, handle), "spc_mailbox_export")
        # the 64-byte IPC handle travels through torch.distributed once per neighbour
        self.hdev = device if (dist.is_initialized() and dist.get_backend() == "nccl") else torch.device("cpu")
        self.handle = torch.frombuffer(bytearray(handle.raw), dtype=torch.uint8).to(self.hdev)
        self.peers = {}       # rank -> (mailbox ptr, data base ptr)
        self.data_top = 0
        self.flag_top = 0

    def _swap(self, mine, rank):
        theirs = torch.empty_like(mine)
        for r in dist.batch_isend_irecv([dist.P2POp(dist.isend, mine, rank), dist.P2POp(dist.irecv, theirs, rank)]):
            r.wait()
        return theirs

    def _peer(self, rank):
        if rank not in self.peers:
            L = _lib.lib()
            raw = bytes(self._swap(self.handle, rank).cpu().numpy().tobytes())
            mb = C.c_void_p()
            _lib.check(L.spc_mailbox_open(C.byref(mb), raw, self.arena_bytes, self.nflags), "spc_mailbox_open")
            self.peers[rank] = (mb, L.spc_mailbox_data(mb))
        return self.peers[rank]

    def _peer_slot(self, slot, rank):
        """(data offset, flag base) of the SAME layer's slot in neighbour `rank`'s arena."""
        ps = slot["peer"]
        if rank not in ps:
            mine = torch.tensor([slot["data"], slot["flags"], slot["slot_bytes"]], dtype=torch.int64, device=self.hdev)
            data, flags, nbytes = [int(v) for v in self._swap(mine, rank).cpu().tolist()]
            if nbytes != slot["slot_bytes"]:
                raise _lib.SpconvError("halo slot mismatch with rank %d: %d vs %d bytes -- the two ranks are not "
                                       "exchanging for the same layer" % (rank, nbytes, slot["slot_bytes"]))
            ps[rank] = (data, flags)
        return ps[rank]

    def _slot(self, layer, x, hh, hw):
        return self._slot_for(layer, (tuple(x.shape), x.dtype, hh, hw), tuple(x.shape), x.element_size(), hh, hw)

    def _slot_for(self, layer, key, shape, esize, hh, hw):
        slots = layer.__dict__.setdefault("_halo_slots", {})
        if key not in slots:
            N, Cc, H, W = shape
            off, offs = 0, []
            for i in range(9):
                offs.append(off)
                if i != 4:
                    n = 1
                    for s in strip_shape(i, N, Cc, H, W, hh, hw):
                        n *= s
                    off += (n * esize + 255) & ~255
            slot_bytes = off
            if self.data_top + 2 * slot_bytes > self.arena_bytes or self.flag_top + self.FLAGS_PER_LAYER > self.nflags:
                raise _lib.SpconvError("halo mailbox arena exhausted; raise SPCONV_ARENA_MB")
            slots[key] = dict(data=self.data_top, flags=self.flag_top, offs=offs, slot_bytes=slot_bytes, peer={}, plan=None,
                              esize=esize)
            self.data_top += 2 * slot_bytes
            self.flag_top += self.FLAGS_PER_LAYER
        return slots[key]

    def _plan(self, slot, shape, hh, hw, mask, ranks):
        """Argument arrays of the two protocol kernels: fixed per (layer, shape, neighbours), built once."""
        key = (tuple(mask), tuple(ranks))
        if slot["plan"] is not None and slot["plan"]["key"] == key:
            return slot["plan"]
        dirs = [i for i in range(9) if i != 4 and mask[i]]
        fb = slot["flags"]
        N, Cc, H, W = shape
        P9, I9, S9 = C.c_void_p * 9, C.c_int * 9, C.c_size_t * 9
        pl = dict(key=key, dirs=dirs, send=P9(), peers=P9(), src=P9(), nbytes=S9(), ack_local=I9(), arr_peer=I9(),
                  arr_local=I9(), ack_peer=I9(), shapes={})
        for d in dirs:
            pmb, pbase = self._peer(ranks[d])
            pdata, pfb = self._peer_slot(slot, ranks[d])
            pl["peers"][d] = pmb
            pl["send"][d] = pbase + pdata + slot["offs"][8 - d]     # my strip d is the neighbour's strip 8-d
            pl["ack_local"][d] = fb + 18 + d                          # neighbour acks what I wrote (my flag)
            pl["arr_peer"][d] = pfb + (8 - d)                         # I announce it on the neighbour's flag
            pl["arr_local"][d] = fb + d                               # neighbour announces my strip d here
            pl["ack_peer"][d] = pfb + 18 + (8 - d)                    # and I ack on its flag
            pl["src"][d] = self.base + slot["data"] + slot["offs"][d]
            shp = strip_shape(d, N, Cc, H, W, hh, hw)
            n = 1
            for s_ in shp:
                n *= s_
            pl["shapes"][d] = shp
            pl["nbytes"][d] = n * slot["esize"]
        slot["plan"] = pl
        return pl

    def exchange(self, layer, x, hh, hw, mask, ranks):
        """Two kernels per exchange: spc_halo_post_auto (wait acks -> pack into the neighbours' slots ->
        signal) and spc_halo_collect_auto (wait arrivals -> copy the strips out -> ack -> advance the
        slot's device-side sequence number).  Nothing in the launch arguments changes from call to call
        except the tile pointer and the receive buffers, so the exchange can be captured in a CUDA graph."""
        L = _lib.lib()
        st = _stream()
        slot = self._slot(layer, x, hh, hw)
        pl = self._plan(slot, x.shape, hh, hw, mask, ranks)
        fb = slot["flags"]
        N, Cc, H, W = x.shape
        dst = (C.c_void_p * 9)()
        recv = [None] * 9
        for d in pl["dirs"]:
            recv[d] = torch.empty(pl["shapes"][d], dtype=x.dtype, device=x.device)
            dst[d] = recv[d].data_ptr()
        _lib.check(L.spc_halo_post_auto(N, Cc, H, W, hh, hw, _lib.dtype_code(x.dtype), C.c_void_p(x.data_ptr()),
                                        C.byref(pl["send"]), slot["slot_bytes"], self.mb, C.byref(pl["peers"]),
                                        C.byref(pl["ack_local"]), C.byref(pl["arr_peer"]), fb + self._SEQ,
                                        fb + self._CNT_POST, st), "spc_halo_post_auto")
        _lib.check(L.spc_halo_collect_auto(C.byref(dst), C.byref(pl["src"]), C.byref(pl["nbytes"]), slot["slot_bytes"],
                                           self.mb, C.byref(pl["peers"]), C.byref(pl["arr_local"]), C.byref(pl["ack_peer"]),
                                           fb + self._SEQ, fb + self._CNT_COLLECT, st), "spc_halo_collect_auto")
        return recv

    def reverse(self, layer, grads, shape, hh, hw, mask, ranks):
        """Reverse exchange of the exact backward (see DistTransport.reverse).  The layer gets a second slot for it,
        fp32-sized, with its own flag block and sequence word, so forward and reverse exchanges of one layer may
        interleave freely; its offsets are swapped with each neighbour at first use like the forward slot's.
        spc_halo_post_strips_auto copies grads[d] into neighbour d's reverse slot, spc_halo_collect_auto copies
        what the neighbours wrote out of this rank's.  Graph-capturable like exchange()."""
        L = _lib.lib()
        st = _stream()
        shape = tuple(shape)
        slot = self._slot_for(layer, ("reverse", shape, hh, hw), shape, 4, hh, hw)
        pl = self._plan(slot, shape, hh, hw, mask, ranks)
        fb = slot["flags"]
        src = (C.c_void_p * 9)()
        dst = (C.c_void_p * 9)()
        recv = [None] * 9
        for d in pl["dirs"]:
            src[d] = grads[d].data_ptr()
            recv[d] = torch.empty(pl["shapes"][d], dtype=torch.float32, device=grads[d].device)
            dst[d] = recv[d].data_ptr()
        _lib.check(L.spc_halo_post_strips_auto(C.byref(src), C.byref(pl["nbytes"]), C.byref(pl["send"]), slot["slot_bytes"],
                                               self.mb, C.byref(pl["peers"]), C.byref(pl["ack_local"]),
                                               C.byref(pl["arr_peer"]), fb + self._SEQ, fb + self._CNT_POST, st),
                   "spc_halo_post_strips_auto")
        _lib.check(L.spc_halo_collect_auto(C.byref(dst), C.byref(pl["src"]), C.byref(pl["nbytes"]), slot["slot_bytes"],
                                           self.mb, C.byref(pl["peers"]), C.byref(pl["arr_local"]), C.byref(pl["ack_peer"]),
                                           fb + self._SEQ, fb + self._CNT_COLLECT, st), "spc_halo_collect_auto")
        return recv

    def arena_high_water(self):
        """Bytes of the mailbox arena handed out to slots so far."""
        return self.data_top


_transport = None


def _single_host_by_env():
    """Rank-independent evidence (no communication): torchrun exports LOCAL_WORLD_SIZE on every rank."""
    try:
        return int(os.environ.get("LOCAL_WORLD_SIZE", "0")) >= int(os.environ.get("WORLD_SIZE", "1"))
    except ValueError:
        return True


def negotiate(device, group=None):
    """COLLECTIVE over `group` (default: the world): decide the halo transport for this job.  The mailbox
    transport needs every rank on ONE host (CUDA IPC) with a working cudaMalloc + IPC export; if any rank
    cannot, ALL ranks take DistTransport (a mixed choice would deadlock).  Called by MPIComm.__init__ (every
    rank constructs it) and bench.py; SPCONV_HALO_TRANSPORT=peer|dist skips the vote."""
    global _transport
    import socket

    kind = os.environ.get("SPCONV_HALO_TRANSPORT", "auto")
    if _transport is not None or device.type != "cuda" or kind != "auto":
        return get_transport(device)
    ok, tr, why = 1, None, ""
    try:
        tr = PeerTransport(device)
    except Exception as e:  # noqa: BLE001 -- any failure means "not on this rank"
        ok, why = 0, str(e)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        try:
            boot = open("/proc/sys/kernel/random/boot_id").read().strip()
        except OSError:
            boot = ""
        idents = [None] * dist.get_world_size(group)
        dist.all_gather_object(idents, (socket.gethostname() + "/" + boot, ok, why), group=group)
        hosts = set(i[0] for i in idents)
        if len(hosts) > 1:
            ok, why = 0, "ranks span %d hosts" % len(hosts)
        for _, o, w in idents:
            if not o:
                ok, why = 0, why or w
    if ok:
        _transport = tr
    else:
        if tr is not None:
            _lib.lib().spc_mailbox_destroy(tr.mb)
        import warnings
        warnings.warn("libspconv: peer-memory halo transport unavailable (%s); all ranks use torch.distributed P2P" % why)
        _transport = DistTransport()
    return _transport


def get_transport(device):
    """The job's halo transport.  SPCONV_HALO_TRANSPORT=peer|dist forces one.  If negotiate() has not run
    (layers used without MPIComm), the choice is made WITHOUT communication from evidence every rank sees
    identically: CUDA device and all ranks on this host (torchrun's LOCAL_WORLD_SIZE) -> PeerTransport, else
    DistTransport; a rank whose mailbox cannot be created then raises (it cannot switch alone)."""
    global _transport
    if _transport is None:
        kind = os.environ.get("SPCONV_HALO_TRANSPORT", "auto" if device.type == "cuda" else "dist")
        if kind == "auto":
            kind = "peer" if _single_host_by_env() else "dist"
        if kind == "peer":
            try:
                _transport = PeerTransport(device)
            except Exception as e:
                raise _lib.SpconvError("peer-memory halo transport could not be set up on this rank (%s); run all ranks "
                                       "with SPCONV_HALO_TRANSPORT=dist, or construct MPIComm / call "
                                       "halo_transport.negotiate() so the ranks agree on the fallback" % e) from e
        else:
            _transport = DistTransport()
    return _transport


def overlap_enabled():
    """Overlap the exchange (comm stream) with the interior pass; SPCONV_HALO_OVERLAP=0 serialises."""
    return os.environ.get("SPCONV_HALO_OVERLAP", "1") != "0"


def exact_backward_default():
    """Initial value of a spatial layer's `exact_backward`: SPCONV_EXACT_BACKWARD=1 sends the gradients of the
    received halo strips back to the neighbours, so that the tiles' input gradients equal the unsplit image's."""
    return os.environ.get("SPCONV_EXACT_BACKWARD", "0") == "1"


def set_transport(t):
    global _transport
    _transport = t
