"""Device engine: the layer between the estimator (L4/L3) and the C-ABI kernels.

It replaces, on the KMeans path only, what the reference delegates to dask (L2 blocked-array
graph + L0 scheduler): row chunks live resident in HBM as torch tensors, each Lloyd iteration
is one fused kernel launch per chunk (``bkm_lloyd_chunk``), and the per-iteration "collective"
— which the reference performs as a task-graph fold plus a client round trip,
dask_ml/cluster/k_means.py:545-552 — is ONE all-reduce of ``[k*d sums | k counts | inertia]``
over ``torch.distributed`` (NCCL on GPUs).

One process drives one GPU.  With ``torch.distributed`` initialised each rank holds its own row
chunks; without it the engine is single-GPU.
"""
import ctypes
import os
import weakref

import numpy as np
import torch

from . import _lib
from .chunked import ChunkedArray, block_dtype, _is_torch

_NP_TO_TORCH = {np.dtype("float32"): torch.float32, np.dtype("float64"): torch.float64}
_DT_CODE = {torch.float32: _lib.BKM_F32, torch.float64: _lib.BKM_F64, torch.bfloat16: _lib.BKM_BF16}


def out_dtype(x_dtype):
    """dtype of the per-row distance outputs for rows of ``x_dtype`` (bf16 rows give float32 distances)."""
    return torch.float32 if x_dtype == torch.bfloat16 else x_dtype


def dist_info():
    """(rank, world_size) of the default process group, (0, 1) when not distributed."""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


class Comm(object):
    """The path's only collective: sum all-reduce (plus tiny object gathers for the init)."""

    def __init__(self):
        self.rank, self.world = dist_info()

    def allreduce_sum_(self, t):
        if self.world > 1:
            p2p = _p2p_state(self) if (t.is_cuda and t.dtype == torch.float64 and t.is_contiguous()) else None
            if p2p is not None and t.numel() <= p2p.max_elems:
                p2p.allreduce_(t)             # one kernel over NVLink peer memory, sums added in rank order
                return t
            import torch.distributed as dist

            dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return t

    def allgather_obj(self, obj):
        if self.world == 1:
            return [obj]
        import torch.distributed as dist

        out = [None] * self.world
        dist.all_gather_object(out, obj)
        return out

    def bcast_obj(self, obj, src=0):
        if self.world == 1:
            return obj
        import torch.distributed as dist

        box = [obj]
        dist.broadcast_object_list(box, src=src)
        return box[0]


class _P2PAllReduce(object):
    """The Lloyd loop's per-iteration collective over NVLink peer memory (bkm_p2p.cu): every rank owns a mailbox that all
    peers of the node have opened through CUDA IPC.  Built once per process (collectively, on first use); any failure —
    ranks on different hosts, IPC unavailable, BKM_P2P=0 — leaves NCCL in charge."""

    MAX_ELEMS = 1 << 16          # float64 elements per slot: k*d + k + 1 of every shape of the fused kernels

    def __init__(self, comm, device):
        import socket

        self.lib = _lib.load()
        self.rank, self.world = comm.rank, comm.world
        self.device = device
        self.max_elems = self.MAX_ELEMS
        self.seq = 0
        self.box = ctypes.c_void_p(0)
        self.peers = []
        ok = os.environ.get("BKM_P2P", "1") != "0" and self.world <= 64
        hosts = comm.allgather_obj(socket.gethostname())
        ok = ok and len(set(hosts)) == 1
        handle = None
        if ok:
            try:
                with torch.cuda.device(device):
                    nb = ctypes.c_size_t(0)
                    _lib.check(self.lib.bkm_p2p_mailbox_bytes(self.world, self.max_elems, ctypes.byref(nb)), "bkm_p2p_mailbox_bytes")
                    _lib.check(self.lib.bkm_p2p_alloc(nb, ctypes.byref(self.box)), "bkm_p2p_alloc")
                    buf = ctypes.create_string_buffer(64)
                    _lib.check(self.lib.bkm_p2p_export(self.box, buf), "bkm_p2p_export")
                    handle = bytes(buf.raw)
            except Exception:
                handle = None
        handles = comm.allgather_obj(handle)                     # collective even when this rank failed
        ptrs = []
        good = all(h is not None for h in handles)
        if good:
            try:
                with torch.cuda.device(device):
                    for r, h in enumerate(handles):
                        if r == self.rank:
                            ptrs.append(int(self.box.value))
                        else:
                            pp = ctypes.c_void_p(0)
                            _lib.check(self.lib.bkm_p2p_import(ctypes.create_string_buffer(h, 64), ctypes.byref(pp)), "bkm_p2p_import")
                            self.peers.append(pp)
                            ptrs.append(int(pp.value))
            except Exception:
                good = False
        self.ready = all(comm.allgather_obj(bool(good)))         # everyone or no one
        if self.ready:
            self.table = torch.tensor(ptrs, dtype=torch.int64, device=device)
            import atexit

            atexit.register(self.close)

    def allreduce_(self, t):
        self.seq += 1
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_allreduce_p2p(
                ctypes.c_void_p(t.data_ptr()), t.numel(), ctypes.c_void_p(self.table.data_ptr()), self.rank, self.world,
                self.max_elems, ctypes.c_uint(self.seq & 0xFFFFFFFF),
                ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)), "bkm_allreduce_p2p")

    def close(self):
        try:
            torch.cuda.synchronize(self.device)
            for pp in self.peers:
                self.lib.bkm_p2p_close(pp)
            self.peers = []
            if self.box.value:
                self.lib.bkm_p2p_free(self.box)
                self.box = ctypes.c_void_p(0)
        except Exception:
            pass
        self.ready = False


_P2P = {}


def _p2p_state(comm):
    """The process-wide peer-memory all-reduce of the current CUDA device, or None (set up collectively on first use)."""
    if not torch.cuda.is_available():
        return None
    dev = torch.device("cuda", torch.cuda.current_device())
    st = _P2P.get(dev)
    if st is None:
        st = _P2PAllReduce(comm, dev)
        _P2P[dev] = st
    return st if st.ready else None


class CudaBackend(object):
    """Calls the sm_90a kernels through the C ABI.  Fails loudly without a GPU/library."""

    name = "b200"
    supports_bf16 = True          # bfloat16 rows: large-shape tensor path (bkm_tc2.cu), d <= 128

    def __init__(self, device=None, flags=0):
        if not torch.cuda.is_available():
            raise RuntimeError(
                "dask_ml_b200 needs a CUDA device: the KMeans hot path is sm_90a CUDA only "
                "and has no CPU fallback."
            )
        self.lib = _lib.load()
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        import os

        self.flags = int(flags) | int(os.environ.get("BKM_FLAGS", "0"))   # BKM_FLAGS: debugging aid
        self._ws = {}

    # -- helpers -------------------------------------------------------------------------
    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    @staticmethod
    def _ptr(t):
        return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)

    def _workspace(self, n, d, k, dtype):
        """Scratch for one chunk call (per-CTA partials + the deferred-row list, 4 bytes per row)."""
        # one grow-only buffer for every shape: the layout inside it is recomputed by the library per call, and
        # k-means|| changes k every round (a buffer per k would allocate ~100 MB per round and keep them all)
        ws = self._ws.get("buf")
        nbytes = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_workspace_bytes(int(n), d, k, _DT_CODE[dtype], ctypes.byref(nbytes)),
                   "bkm_workspace_bytes")
        if ws is None or ws.numel() < nbytes.value:
            ws = torch.empty(int(nbytes.value * 1.25) + (1 << 20), dtype=torch.uint8, device=self.device)
            ws[:8192].zero_()        # the persistent header (balance table of the M-step row pass) starts out empty
            self._ws["buf"] = ws
        return ws

    def kernel_family(self, d, k, dtype):
        return self.lib.bkm_kernel_family(d, k, _DT_CODE[dtype], self.flags)

    def launch_count(self):
        return int(self.lib.bkm_launch_count())

    _fallbacks_seen = 0

    def _note_fallback(self, x):
        """Warn (once per process) when a chunk whose shape belongs to the tensor / streaming kernels ran on the generic
        CUDA-core kernel because its rows are not 16-byte aligned — results are identical, throughput is not."""
        c = int(self.lib.bkm_debug_fallback_count())
        if c != CudaBackend._fallbacks_seen:
            first = CudaBackend._fallbacks_seen == 0
            CudaBackend._fallbacks_seen = c
            if first:
                import warnings
                warnings.warn("dask_ml_b200: a chunk with shape %s, row pitch %d elements, base address %% 16 = %d is not "
                              "16-byte aligned; the generic CUDA-core kernel is used instead of the tensor-core / streaming "
                              "kernel (pass the data through CudaBackend.to_device, which pads the row pitch)"
                              % (tuple(x.shape), x.stride(0), x.data_ptr() % 16), RuntimeWarning, stacklevel=3)

    def abort_code(self):
        """Non-zero once a pipeline wait of the tensor kernel has timed out (synchronises the device)."""
        return int(self.lib.bkm_debug_abort_code())

    def reset_abort(self):
        self.lib.bkm_debug_reset()

    def deferred_rows(self, n, d, k, dtype):
        """Rows the last tensor-path chunk call of this shape handed to the float64 re-check (debug / bench)."""
        ws = self._ws.get("buf")
        if ws is None:
            return None
        c = ctypes.c_int(0)
        _lib.check(self.lib.bkm_debug_deferred_rows(self._ptr(ws), int(n), d, k, _DT_CODE[dtype], ctypes.byref(c)),
                   "bkm_debug_deferred_rows")
        return int(c.value)

    # -- data ----------------------------------------------------------------------------
    def to_device(self, block, dtype):
        """numpy / torch block -> contiguous CUDA tensor of `dtype` (torch dtype)."""
        if _is_torch(block):
            t = block
        else:
            a = np.ascontiguousarray(block)
            if not a.flags.writeable:
                a = a.copy()                 # torch refuses read-only buffers
            t = torch.from_numpy(a)
        t = t.to(device=self.device, dtype=dtype, non_blocking=True)
        if t.dim() == 2 and dtype == torch.bfloat16 and t.shape[0] > 0 and (t.shape[1] % 8 or t.stride(0) % 8 or t.stride(1) != 1):
            # bf16 rows are read by TMA: 16-byte row pitch = a multiple of 8 elements (zero padded view)
            n, d = t.shape
            buf = torch.zeros((n, (d + 7) // 8 * 8), dtype=dtype, device=self.device)
            buf[:, :d] = t
            return buf[:, :d]
        if t.dim() == 2 and dtype == torch.bfloat16:
            return t
        if t.dim() == 2 and dtype == torch.float32 and t.shape[1] % 4 and t.shape[1] <= 64 and t.shape[0] > 0:
            # The tensor path reads row tiles with TMA, which needs a 16-byte row pitch: rows are stored with the
            # pitch rounded up to 4 floats (zero padded) and handed on as a (n, d) view of that buffer.
            n, d = t.shape
            buf = torch.zeros((n, (d + 3) // 4 * 4), dtype=dtype, device=self.device)
            buf[:, :d] = t
            return buf[:, :d]
        return t.contiguous()

    def empty(self, shape, dtype):
        return torch.empty(shape, dtype=dtype, device=self.device)

    def zeros(self, shape, dtype):
        return torch.zeros(shape, dtype=dtype, device=self.device)

    # -- kernels -------------------------------------------------------------------------
    def check_finite(self, chunks):
        flag = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            for x in chunks:
                n, d = x.shape
                _lib.check(self.lib.bkm_check_finite(self._ptr(x), n, d, x.stride(0), _DT_CODE[x.dtype],
                                                     self._ptr(flag), self._stream()), "bkm_check_finite")
        return flag

    def pack_centers(self, C64, dtype, out=None):
        k, d = C64.shape
        nbytes = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_centers_pack_bytes(k, d, _DT_CODE[dtype], ctypes.byref(nbytes)),
                   "bkm_centers_pack_bytes")
        if out is None or out.numel() < nbytes.value:
            out = torch.empty(nbytes.value, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_pack_centers(self._ptr(C64), k, d, _DT_CODE[dtype], self._ptr(out),
                                                 out.numel(), self._stream()), "bkm_pack_centers")
        return out

    def lloyd_chunk(self, x, pack, k, labels, min_d2, sums, counts, inertia, first=False, loop_state=None):
        """Fused E+M step of one chunk.  ``counts`` may be int64 or float64 (one float64 buffer for the all-reduce);
        ``first`` overwrites the accumulators instead of adding (first chunk of an iteration); ``loop_state`` makes
        the call a no-op once the device-side loop has converged."""
        n, d = x.shape
        ws = self._workspace(n, d, k, x.dtype)
        flags = self.flags
        if first:
            flags |= _lib.FLAG_FIRST_CHUNK
        if counts is not None and counts.dtype == torch.float64:
            flags |= _lib.FLAG_COUNTS_F64
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_lloyd_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(pack), k,
                self._ptr(labels), self._ptr(min_d2), self._ptr(sums), self._ptr(counts),
                self._ptr(inertia), self._ptr(ws), ws.numel(), flags, self._ptr(loop_state), self._stream()),
                "bkm_lloyd_chunk")
        self._note_fallback(x)

    # -- device-resident Lloyd loop ------------------------------------------------------
    def loop_state_new(self, tol, max_iter):
        """(state bytes, shift history) for one Lloyd loop, reset on the device."""
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_loop_state_bytes(ctypes.byref(nb)), "bkm_loop_state_bytes")
        state = torch.zeros(int(nb.value), dtype=torch.uint8, device=self.device)
        hist = torch.zeros(max(1, int(max_iter)), dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_loop_reset(self._ptr(state), float(tol), self._ptr(hist), int(hist.numel()),
                                               self._stream()), "bkm_loop_reset")
        return state, hist

    def loop_state_read(self, state):
        """(done, n_iter, shift) — one device->host copy (the loop's only synchronisation)."""
        raw = state.cpu().numpy()
        done, n_iter = np.frombuffer(raw[:8].tobytes(), dtype=np.int32)
        shift = np.frombuffer(raw[24:32].tobytes(), dtype=np.float64)[0]
        return int(done), int(n_iter), float(shift)

    def finalize_step(self, red, c_in, c_out, state, pack, dtype):
        k, d = c_in.shape
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_finalize_step(self._ptr(red), self._ptr(c_in), self._ptr(c_out), self._ptr(state),
                                                  k, d, _DT_CODE[dtype], self._ptr(pack), pack.numel(), self._stream()),
                       "bkm_finalize_step")

    def minibatch_step(self, red, c_in, w_in, c_out, w_out, pack, dtype):
        """One mini-batch centre update from ``red = [k*d sums | k counts | inertia]`` of the batch: c_out, w_out and the
        pack of c_out (scikit-learn's _minibatch_update_dense, in float64)."""
        k, d = c_in.shape
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_minibatch_step(self._ptr(red), self._ptr(c_in), self._ptr(w_in), self._ptr(c_out),
                                                   self._ptr(w_out), k, d, _DT_CODE[dtype], self._ptr(pack), pack.numel(),
                                                   self._stream()), "bkm_minibatch_step")

    def assign_chunk(self, x, pack, k, labels, min_dist, squared, dist_sum):
        n, d = x.shape
        ws = self._workspace(n, d, k, x.dtype)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_assign_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(pack), k,
                self._ptr(labels), self._ptr(min_dist), int(bool(squared)), self._ptr(dist_sum),
                self._ptr(ws), ws.numel(), self.flags, self._stream()), "bkm_assign_chunk")
        self._note_fallback(x)

    def sample_chunk(self, min_d2, ell_over_phi, seed, row_offset, picked, n_picked):
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_sample_chunk(
                self._ptr(min_d2), min_d2.numel(), _DT_CODE[min_d2.dtype], float(ell_over_phi),
                int(seed) & 0xFFFFFFFFFFFFFFFF, int(row_offset), self._ptr(picked), picked.numel(),
                self._ptr(n_picked), self._stream()), "bkm_sample_chunk")

    def min_fold(self, run_min, new_min, phi_acc):
        """run_min = min(run_min, new_min) (new_min may be None) and phi_acc += sum(run_min): one kernel."""
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_min_fold_chunk(self._ptr(run_min), self._ptr(new_min), run_min.numel(),
                                                   _DT_CODE[run_min.dtype], self._ptr(phi_acc), self._stream()),
                       "bkm_min_fold_chunk")

    def transform_chunk(self, x, pack, k, out, mode=0, gamma=0.0):
        """(n, k) block of distances (mode 0), squared distances (1) or exp(-gamma d^2) (2) into ``out`` — which may be a
        column block of a wider matrix (row pitch = out.stride(0))."""
        n, d = x.shape
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_transform_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(pack), k,
                self._ptr(out), out.stride(0) if n else k, int(mode), float(gamma), self.flags, self._stream()),
                "bkm_transform_chunk")

    def kernel_colsum(self, x, pack, l, gamma, colsum, first=False):
        """colsum[j] (+)= sum_i exp(-gamma ||x_i - c_j||^2) over the rows of the chunk (float64 [l]); ``first`` overwrites.
        The first pass of the Nystrom embedding (SpectralClustering)."""
        n, d = x.shape
        ws = self._workspace(n, d, l, x.dtype)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_kernel_colsum_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(pack), int(l), float(gamma),
                self._ptr(colsum), self._ptr(ws), ws.numel(), flags, self._stream()), "bkm_kernel_colsum_chunk")

    def nystrom_embed(self, x, pack, l, gamma, W, out):
        """out[i] = e_i / ||e_i||, e_i = sum_j exp(-gamma (||x_i - c_j||^2 - min_j ||x_i - c_j||^2)) W[j] — the second
        pass of the Nystrom embedding.  ``W`` is (l, k) in the dtype of x; ``out`` (n, k) may have a padded row pitch."""
        n, d = x.shape
        k = int(W.shape[1])
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_nystrom_embed_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(pack), int(l), float(gamma),
                self._ptr(W), k, self._ptr(out), out.stride(0) if n else k, self.flags, self._stream()),
                "bkm_nystrom_embed_chunk")

    def finalize(self, sums, counts, C_old, C_new, shift):
        k, d = C_old.shape
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_finalize(self._ptr(sums), self._ptr(counts), self._ptr(C_old),
                                             self._ptr(C_new), self._ptr(shift), k, d, self._stream()),
                       "bkm_finalize")


def _host_unregister(tensors):
    """End the page-lock registrations made by ``StreamedChunks`` (runs when it is collected or at interpreter exit,
    while the tensors — and so the memory — are still alive)."""
    try:
        rt = torch.cuda.cudart()
        torch.cuda.synchronize()                   # no copy may still read the pages
        for t in tensors:
            rt.cudaHostUnregister(t.data_ptr())
    except Exception:
        pass
    del tensors[:]


class StreamedChunks(object):
    """Row chunks that stay in HOST memory and pass through two device buffers every time they are iterated: the
    out-of-core ingestion path (data larger than HBM, or simply not uploaded).  Iterating yields device tensors in
    order; block i+1 is copied host->device on a copy stream while the kernels enqueued for block i run, so X crosses
    PCIe once per sweep.  A yielded tensor is valid until the iterator is advanced (its buffer is then recycled)."""

    def __init__(self, host_blocks, backend, dtype, block_rows=1 << 20):
        self.backend = backend
        self.dtype = dtype
        self.parts = []                            # (host tensor view of <= block_rows rows)
        registered = []                            # host tensors page-locked here (kept alive until unregistered)
        self._unpin = weakref.finalize(self, _host_unregister, registered)
        for b in host_blocks:
            t = b if _is_torch(b) else torch.from_numpy(np.ascontiguousarray(b))
            t = t.to(dtype) if t.dtype != dtype else t
            if not t.is_contiguous():
                t = t.contiguous()
            if backend.device.type == "cuda" and not t.is_pinned() and t.numel() > 0:
                # page-lock in place (no second host copy): asynchronous H2D copies need pinned memory.  The
                # registration MUST end before the memory is released: a stale registration of a recycled address
                # range makes later device->host copies of unrelated tensors land in the wrong pages.
                try:
                    rc = torch.cuda.cudart().cudaHostRegister(t.data_ptr(), t.numel() * t.element_size(), 0)
                except Exception:
                    rc = 1
                if int(rc) == 0:
                    registered.append(t)
            for s0 in range(0, max(1, int(t.shape[0])), block_rows):
                self.parts.append(t[s0:s0 + block_rows])
        self.sizes = [int(p.shape[0]) for p in self.parts]
        self.d = int(self.parts[0].shape[1])
        self._bufs = None

    def __len__(self):
        return len(self.parts)

    def __iter__(self):
        return self.iter_order(range(len(self.parts)))

    def iter_order(self, order):
        """Iterate the parts in ``order`` (a sequence of part indices), with the same double buffering."""
        be = self.backend
        if be.device.type != "cuda":
            for i in order:
                yield self.parts[i]
            return
        if self._bufs is None:
            rows = max(self.sizes) if self.sizes else 1
            pitch = self.d
            if self.dtype == torch.float32 and self.d % 4 and self.d <= 64:
                pitch = (self.d + 3) // 4 * 4          # 16-byte rows for the tensor path (see CudaBackend.to_device)
            if self.dtype == torch.bfloat16 and self.d % 8:
                pitch = (self.d + 7) // 8 * 8
            self._bufs = [torch.zeros((max(1, rows), pitch), dtype=self.dtype, device=be.device) for _ in range(2)]
            self._copy_stream = torch.cuda.Stream(device=be.device)
        main = torch.cuda.current_stream(be.device)
        consumed = [None, None]
        for pos, i in enumerate(order):
            p = self.parts[i]
            slot = pos & 1
            m = int(p.shape[0])
            with torch.cuda.stream(self._copy_stream):
                if consumed[slot] is not None:
                    self._copy_stream.wait_event(consumed[slot])
                else:
                    self._copy_stream.wait_stream(main)       # a previous sweep may still read this buffer
                self._bufs[slot][:m, :self.d].copy_(p, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self._copy_stream)
            main.wait_event(ev)
            yield self._bufs[slot][:m, :self.d]
            done = torch.cuda.Event()
            done.record(main)
            consumed[slot] = done

    def __getitem__(self, i):
        raise TypeError("streamed chunks cannot be indexed; iterate them")


class DeviceData(object):
    """Row chunks of X + their place in the global (all-rank) row order.  The chunks are resident on the device
    (list of tensors) or, for ``HostData``, streamed from host memory on every sweep (``StreamedChunks``)."""

    def __init__(self, chunks, backend, comm=None):
        self.chunks = chunks                      # list of 2-D torch tensors on backend.device (or StreamedChunks)
        self.backend = backend
        self.comm = comm or Comm()
        if isinstance(chunks, StreamedChunks):
            self.dtype, self.d = chunks.dtype, chunks.d
            self.chunk_rows = list(chunks.sizes)
        else:
            self.dtype = chunks[0].dtype
            self.d = int(chunks[0].shape[1])
            self.chunk_rows = [int(c.shape[0]) for c in chunks]
        self._init_layout()

    def _init_layout(self):
        chunks = self.chunks
        self.n_local = int(sum(self.chunk_rows))
        sizes = self.comm.allgather_obj(self.n_local)
        self.rank_sizes = [int(s) for s in sizes]
        self.row_offset = int(sum(self.rank_sizes[: self.comm.rank]))
        self.n_global = int(sum(self.rank_sizes))
        self.chunk_offsets = np.cumsum([0] + list(self.chunk_rows))

    @property
    def np_dtype(self):
        """dtype of host-side results (cluster_centers_): that of X; float32 for bfloat16 rows (numpy has no bf16)."""
        return np.dtype("float64") if self.dtype == torch.float64 else np.dtype("float32")

    @property
    def out_dtype(self):
        return out_dtype(self.dtype)

    def local_rows(self, local_idx):
        """Rows by LOCAL index -> numpy (len, d)."""
        local_idx = np.asarray(local_idx, dtype=np.int64)
        out = np.empty((len(local_idx), self.d), dtype=self.np_dtype)
        if isinstance(self.chunks, StreamedChunks):
            which = np.searchsorted(self.chunk_offsets, local_idx, side="right") - 1
            for w in np.unique(which):
                pos = np.nonzero(which == w)[0]
                part = self.chunks.parts[w]
                sel = part[torch.as_tensor(local_idx[pos] - self.chunk_offsets[w], dtype=torch.int64)]
                out[pos] = (sel.float() if sel.dtype == torch.bfloat16 else sel).numpy()
            return out
        which = np.searchsorted(self.chunk_offsets, local_idx, side="right") - 1
        # one gather + one device-to-host copy per chunk that holds requested rows (not one copy per row)
        for w in np.unique(which):
            pos = np.nonzero(which == w)[0]
            rel = torch.as_tensor(local_idx[pos] - self.chunk_offsets[w], dtype=torch.int64, device=self.chunks[w].device)
            sel = self.chunks[w].index_select(0, rel)
            out[pos] = (sel.float() if sel.dtype == torch.bfloat16 else sel).cpu().numpy()
        return out

    def global_rows(self, global_idx):
        """Rows by GLOBAL index (any rank's rows), returned on every rank in the given order."""
        global_idx = np.asarray(global_idx, dtype=np.int64)
        lo, hi = self.row_offset, self.row_offset + self.n_local
        mine = np.nonzero((global_idx >= lo) & (global_idx < hi))[0]
        rows = self.local_rows(global_idx[mine] - lo)
        if self.comm.world == 1:
            return rows
        parts = self.comm.allgather_obj((mine, rows))
        out = np.empty((len(global_idx), self.d), dtype=self.np_dtype)
        for pos, r in parts:
            out[pos] = r
        return out

    def to_host(self):
        """All LOCAL rows as one numpy array (used only by the in-memory k-means++ init)."""
        src = self.chunks.parts if isinstance(self.chunks, StreamedChunks) else self.chunks
        return np.concatenate([(c.float() if c.dtype == torch.bfloat16 else c).cpu().numpy() for c in src], axis=0)


def host_resident(X, backend=None, comm=None, block_rows=1 << 20):
    """Wrap host-resident data (ndarray / CPU tensor / ChunkedArray of host blocks) for OUT-OF-CORE use: ``KMeans.fit``,
    ``predict`` and the metrics then stream the rows through two device buffers on every sweep instead of uploading X
    (``StreamedChunks``).  Use it for data larger than HBM; everything else is unchanged (same kernels, same results)."""
    from .chunked import ChunkedArray as _CA

    backend = backend or CudaBackend()
    blocks = X.blocks if isinstance(X, _CA) else [X]
    first = blocks[0]
    if _is_torch(first):
        dt = first.dtype if first.dtype in (torch.float32, torch.float64, torch.bfloat16) else torch.float64
    else:
        nd = np.dtype(first.dtype)
        dt = torch.float32 if nd in (np.dtype("float32"), np.dtype("int32"), np.dtype("float16")) else torch.float64
    return DeviceData(StreamedChunks(blocks, backend, dt, block_rows), backend, comm)
