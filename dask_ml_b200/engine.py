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
_METRIC_CODE = {**_DT_CODE, torch.float16: _lib.BKM_M_F16, torch.int32: _lib.BKM_M_I32, torch.int64: _lib.BKM_M_I64,
                torch.bool: _lib.BKM_M_U8, torch.uint8: _lib.BKM_M_U8}
# element types of the encoders' passes (X, one-hot outputs and codes)
_ENC_CODE = {torch.float32: _lib.BKM_F32, torch.float64: _lib.BKM_F64, torch.bfloat16: _lib.BKM_BF16,
             torch.int32: _lib.BKM_M_I32, torch.int64: _lib.BKM_M_I64, torch.bool: _lib.BKM_M_U8,
             torch.uint8: _lib.BKM_M_U8}


def out_dtype(x_dtype):
    """dtype of the per-row distance outputs for rows of ``x_dtype`` (bf16 rows give float32 distances)."""
    return torch.float32 if x_dtype == torch.bfloat16 else x_dtype


def dist_info():
    """(rank, world_size) of the default process group, (0, 1) when not distributed."""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def single_process(who):
    """Raise NotImplementedError under torch.distributed with more than one rank, for the estimators that visit the
    blocks one after another in one process.  Called before anything that could be a collective, so that every rank
    raises instead of waiting for the others."""
    world = dist_info()[1]
    if world > 1:
        raise NotImplementedError("%s steps through the blocks one after another in one process; it does not run "
                                  "under torch.distributed (world size %d)" % (who, world))


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

    def _scratch(self, key, nbytes):
        """A grow-only device buffer of at least ``nbytes`` per key (the workspace of one kind of pass)."""
        ws = self._ws.get(key)
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=self.device)
            self._ws[key] = ws
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
            buf = self.rows_buffer(t.shape[0], t.shape[1], dtype)
            buf.copy_(t)
            return buf
        if t.dim() == 2 and dtype == torch.bfloat16:
            return t
        if t.dim() == 2 and dtype == torch.float32 and t.shape[1] % 4 and t.shape[1] <= 64 and t.shape[0] > 0:
            buf = self.rows_buffer(t.shape[0], t.shape[1], dtype)
            buf.copy_(t)
            return buf
        return t.contiguous()

    def rows_buffer(self, n, d, dtype):
        """An (n, d) device block with the row pitch ``to_device`` gives rows of ``dtype``."""
        pitch = d
        if n > 0 and dtype == torch.bfloat16 and d % 8:
            pitch = (d + 7) // 8 * 8             # bf16 rows are read by TMA: a 16-byte row pitch
        elif n > 0 and dtype == torch.float32 and d % 4 and d <= 64:
            # The tensor path reads row tiles with TMA, which needs a 16-byte row pitch: rows are stored with the
            # pitch rounded up to 4 floats (zero padded) and handed on as a (n, d) view of that buffer.
            pitch = (d + 3) // 4 * 4
        if pitch == d:
            return torch.empty((n, d), dtype=dtype, device=self.device)
        return torch.zeros((n, pitch), dtype=dtype, device=self.device)[:, :d]

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

    def gram_chunk(self, x, shift, colsum, gram, first=False):
        """colsum (+)= sum_i (x_i - shift) and gram (+)= sum_i (x_i - shift)(x_i - shift)^T over the rows of the chunk
        (float64 [d] and [d, d] on the device); ``first`` overwrites.  The fit pass of PCA / TruncatedSVD."""
        n, d = x.shape
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_gram_workspace_bytes(int(n), int(d), ctypes.byref(nb)), "bkm_gram_workspace_bytes")
        ws = self._scratch("gram", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_gram_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(shift), self._ptr(colsum),
                self._ptr(gram), self._ptr(ws), ws.numel(), flags, self._stream()), "bkm_gram_chunk")

    def project_chunk(self, x, shift, W, out=None, colmax=None, row_offset=0):
        """out = (x - shift) W^T (``W`` float64 (k, d), ``shift`` float64 (d,) or None, ``out`` (n, k) float32 / float64
        with any row pitch, or None) and, into ``colmax`` (float64 (k, 4) records, see ``colmax_new``), per column
        the largest |out_ij| with its lowest global row ``row_offset + i`` and its signed value."""
        n, d = x.shape
        k = int(W.shape[0])
        odt = _DT_CODE[out.dtype] if out is not None else _lib.BKM_F64
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_project_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(shift), self._ptr(W), k,
                self._ptr(out), (out.stride(0) if n else k) if out is not None else k, odt, self._ptr(colmax),
                int(row_offset), self.flags, self._stream()), "bkm_project_chunk")

    def colmax_new(self, k):
        """k empty arg-max records {absmax = -1, row = -1, value = 0, lock = 0} for ``project_chunk``."""
        rec = torch.zeros((k, 4), dtype=torch.float64)
        rec[:, 0] = -1.0
        rec[:, 1:2].view(torch.int64).fill_(-1)
        return rec.to(self.device)

    def class_moments_chunk(self, x, cls, K, sums, counts=None, theta=None, first=False):
        """GaussianNB's fit passes over the rows of one chunk, by int32 class index ``cls`` (indices outside [0, K) are
        skipped): without ``theta``, sums (K, d) (+)= per-class row sums and counts (K,) (+)= per-class rows; with
        ``theta`` (float64 (K, d)), sums (+)= per-class sums of (x - theta_c)^2.  float64 on the device; ``first``
        overwrites."""
        n, d = x.shape
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_nb_workspace_bytes(int(n), int(d), int(K), ctypes.byref(nb)), "bkm_nb_workspace_bytes")
        ws = self._scratch("nb", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        mode = 0 if theta is None else 1
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_class_moments_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(cls), int(K), mode,
                self._ptr(theta), self._ptr(sums), self._ptr(counts), self._ptr(ws), ws.numel(), flags,
                self._stream()), "bkm_class_moments_chunk")

    def nb_jll_chunk(self, x, theta, inv_sigma, logc, labels=None, out=None, exp_out=False, n_deferred=None):
        """GaussianNB's predict pass over one chunk: ``labels`` (int32 (n,)) the arg-max of the joint log-likelihood
        and / or ``out`` (float64 (n, K), any row pitch) its log-softmax, exponentiated with ``exp_out``.  ``theta``,
        ``inv_sigma`` float64 (K, d), ``logc`` float64 (K,) on the device; ``n_deferred`` (int32 (1,)) counts the fp32
        rows re-decided in float64."""
        n, d = x.shape
        K = int(theta.shape[0])
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_nb_jll_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(theta), self._ptr(inv_sigma),
                self._ptr(logc), K, self._ptr(labels), self._ptr(out),
                (out.stride(0) if n else K) if out is not None else K, int(bool(exp_out)), self._ptr(n_deferred),
                self.flags, self._stream()), "bkm_nb_jll_chunk")

    def class_counts_chunk(self, x, cls, K, fc, cc, w=None, binarize=None, first=False):
        """The count pass of the discrete naive Bayes models over one chunk, by int32 class index ``cls`` (indices
        outside [0, K) are skipped): fc (K, d) (+)= per-class sums of w_i f(x_i) and cc (K,) (+)= per-class sums of w_i,
        float64 on the device, ``w`` float64 (n,) or None (ones), f(x) = x, or x > ``binarize`` when it is not None.
        ``first`` overwrites."""
        n, d = x.shape
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_nb_workspace_bytes(int(n), int(d), int(K), ctypes.byref(nb)), "bkm_nb_workspace_bytes")
        ws = self._scratch("nb", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_class_counts_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(cls), int(K), self._ptr(w),
                int(binarize is not None), float(binarize or 0.0), self._ptr(fc), self._ptr(cc), self._ptr(ws),
                ws.numel(), flags, self._stream()), "bkm_class_counts_chunk")

    def csc_class_counts_chunk(self, csc, d, labels, K, fcT, w=None, binarize=None, first=False):
        """``class_counts_chunk``'s feature sums over the transpose ``csc`` of one CSR block, transposed: fcT (d, K)
        (+)= per-class sums of w_i f(x_ij), each in ascending row order; an entry not above ``binarize`` adds nothing.
        ``first`` overwrites."""
        colptr, rows, vals, plan = csc
        nnz = int(rows.numel())
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_csc_label_sums_workspace_bytes(int(d), nnz, int(K), ctypes.byref(nb)),
                   "bkm_csc_label_sums_workspace_bytes")
        ws = self._scratch("csc_label_sums", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_csc_class_counts_chunk(
                self._ptr(colptr), self._ptr(rows), self._ptr(vals), _DT_CODE[vals.dtype], int(d), nnz, self._ptr(plan),
                self._ptr(labels), int(K), self._ptr(w), int(binarize is not None), float(binarize or 0.0),
                self._ptr(fcT), self._ptr(ws), ws.numel(), flags, self._stream()), "bkm_csc_class_counts_chunk")

    def nb_linear_jll_chunk(self, x, W, b, labels=None, out=None, out_mode=0, binarize=None):
        """The predict pass of the discrete naive Bayes models over one chunk: jll = f(x) W^T + b (``W`` float64 (K, d),
        ``b`` float64 (K,) on the device; f as in ``class_counts_chunk``), into ``labels`` (int32 (n,)) its arg-max and /
        or ``out`` (float64 (n, K), any row pitch) jll (``out_mode`` 0), its log-softmax (1) or softmax (2)."""
        n, d = x.shape
        K = int(W.shape[0])
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_nb_linear_jll_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], int(binarize is not None),
                float(binarize or 0.0), self._ptr(W), self._ptr(b), K, self._ptr(labels), self._ptr(out),
                (out.stride(0) if n else K) if out is not None else K, int(out_mode), self.flags, self._stream()),
                "bkm_nb_linear_jll_chunk")

    def nb_csr_jll_chunk(self, blk, d, WT, b, labels=None, out=None, out_mode=0, binarize=None):
        """``nb_linear_jll_chunk`` on one CSR block of d columns over its stored entries, ``WT`` float64 (d, K)
        row-major."""
        crow, col, val, n = blk
        K = int(WT.shape[1])
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_nb_csr_jll_chunk(
                self._ptr(crow), self._ptr(col), self._ptr(val), _DT_CODE[val.dtype], int(n), int(d), int(col.numel()),
                int(binarize is not None), float(binarize or 0.0), self._ptr(WT), self._ptr(b), K, self._ptr(labels),
                self._ptr(out), (out.stride(0) if n else K) if out is not None else K, int(out_mode), self.flags,
                self._stream()), "bkm_nb_csr_jll_chunk")

    def glm_pass_chunk(self, x, y, beta, family, mode, grad=None, hrow=None, w=None, out=None, first=False):
        """The fused pass of the linear models over one chunk (float64 arithmetic): eta = x . beta[:d] + beta[d] with
        ``family`` 0 logistic, 1 normal, 2 poisson.  ``mode`` 0: grad (d + 2,) (+)= [sum r x | sum r | loss];
        1: the same, w (n,) = the Newton weights and hrow (d + 1,) (+)= [sum w x | sum w]; 2: out (n,) float64 = mu;
        3: out (n,) uint8 = mu > 0.5.  ``y`` float64 (n,) (modes 0 and 1), ``beta`` float64 (d + 1,) on the device;
        ``first`` overwrites."""
        n, d = x.shape
        ws = None
        if mode in (0, 1):
            nb = ctypes.c_size_t(0)
            _lib.check(self.lib.bkm_glm_workspace_bytes(int(n), int(d), ctypes.byref(nb)), "bkm_glm_workspace_bytes")
            ws = self._scratch("glm", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_glm_pass_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(y), self._ptr(beta),
                int(family), int(mode), self._ptr(grad), self._ptr(hrow), self._ptr(w), self._ptr(out), self._ptr(ws),
                ws.numel() if ws is not None else 0, flags, self._stream()), "bkm_glm_pass_chunk")

    def gram_weighted_chunk(self, x, w, gram, first=False):
        """gram (+)= sum_i w_i x_i x_i^T over the rows of the chunk (``w`` float64 (n,), ``gram`` float64 (d, d) on the
        device): the Hessian block of a Newton step.  ``first`` overwrites."""
        n, d = x.shape
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_gram_workspace_bytes(int(n), int(d), ctypes.byref(nb)), "bkm_gram_workspace_bytes")
        ws = self._scratch("gram", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_gram_weighted_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(w), self._ptr(gram),
                self._ptr(ws), ws.numel(), flags, self._stream()), "bkm_gram_weighted_chunk")

    def glm_csr_pass_chunk(self, blk, d, y, beta, family, mode, r=None, w=None, grad=None, hrow=None, out=None,
                           first=False):
        """``glm_pass_chunk`` on one CSR block ``blk`` = (crow int64 (n + 1,), col int64 (nnz,), val float32 / float64
        (nnz,), n) of d columns.  Modes 0 and 1 write r (n,) (and w (n,)) float64 for ``csc_matvec_chunk`` and set
        grad[d:d + 2] = [sum r | loss] (and hrow[d] = sum w); modes 2 and 3 write ``out`` as the dense pass does."""
        crow, col, val, n = blk
        ws = None
        if mode in (0, 1):
            nb = ctypes.c_size_t(0)
            _lib.check(self.lib.bkm_glm_csr_workspace_bytes(int(n), ctypes.byref(nb)), "bkm_glm_csr_workspace_bytes")
            ws = self._scratch("glm_csr", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_glm_csr_pass_chunk(
                self._ptr(crow), self._ptr(col), self._ptr(val), _DT_CODE[val.dtype], int(n), int(d), int(col.numel()),
                self._ptr(y), self._ptr(beta), int(family), int(mode), self._ptr(r), self._ptr(w), self._ptr(grad),
                self._ptr(hrow), self._ptr(out), self._ptr(ws), ws.numel() if ws is not None else 0, flags,
                self._stream()), "bkm_glm_csr_pass_chunk")

    def csr_transpose_chunk(self, blk, d):
        """The CSC of one CSR block: (colptr int64 (d + 1,), rows int32 (nnz,) ascending within each column, vals
        (nnz,) in the block's dtype, plan int64), plan[:4] = [non-canonical flag | segments | Gram slots | longest
        column] (include/bkm_b200.h)."""
        crow, col, val, n = blk
        nnz = int(col.numel())
        wb, pb = ctypes.c_size_t(0), ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_csr_transpose_workspace_bytes(int(n), int(d), nnz, ctypes.byref(wb), ctypes.byref(pb)),
                   "bkm_csr_transpose_workspace_bytes")
        ws = self._scratch("csr_transpose", wb.value)
        colptr = torch.empty(int(d) + 1, dtype=torch.int64, device=self.device)
        rows = torch.empty(nnz, dtype=torch.int32, device=self.device)
        vals = torch.empty(nnz, dtype=val.dtype, device=self.device)
        plan = torch.empty((pb.value + 7) // 8, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_csr_transpose_chunk(
                self._ptr(crow), self._ptr(col), self._ptr(val), _DT_CODE[val.dtype], int(n), int(d), nnz,
                self._ptr(colptr), self._ptr(rows), self._ptr(vals), self._ptr(plan), plan.numel() * 8, self._ptr(ws),
                ws.numel(), self._stream()), "bkm_csr_transpose_chunk")
        return colptr, rows, vals, plan

    def csc_matvec_chunk(self, csc, d, v1, out1, v2=None, out2=None, first=False):
        """out1[:d] (+)= X^T v1 (and out2[:d] (+)= X^T v2) over the transpose ``csc`` of one block, each column's
        entries added in ascending row order.  ``first`` overwrites."""
        colptr, rows, vals, plan = csc
        nnz = int(rows.numel())
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_csc_matvec_workspace_bytes(int(d), nnz, ctypes.byref(nb)),
                   "bkm_csc_matvec_workspace_bytes")
        ws = self._scratch("csc_matvec", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_csc_matvec_chunk(
                self._ptr(colptr), self._ptr(rows), self._ptr(vals), _DT_CODE[vals.dtype], int(d), nnz, self._ptr(plan),
                self._ptr(v1), self._ptr(v2), self._ptr(out1), self._ptr(out2), self._ptr(ws), ws.numel(), flags,
                self._stream()), "bkm_csc_matvec_chunk")

    def gram_weighted_csr_chunk(self, blk, csc, d, w, gram, n_slots, first=False):
        """gram (d, d) (+)= sum_i w_i x_i x_i^T over one CSR block and its transpose; ``n_slots`` = plan[2] of the
        transpose (read once per fit).  ``first`` overwrites."""
        crow, col, val, n = blk
        colptr, rows, vals, plan = csc
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_gram_weighted_csr_workspace_bytes(int(d), int(n_slots), ctypes.byref(nb)),
                   "bkm_gram_weighted_csr_workspace_bytes")
        ws = self._scratch("gram_csr", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_gram_weighted_csr_chunk(
                self._ptr(crow), self._ptr(col), self._ptr(val), _DT_CODE[val.dtype], int(n), int(d),
                int(col.numel()), self._ptr(colptr), self._ptr(rows), self._ptr(vals), self._ptr(plan), int(n_slots),
                self._ptr(w), self._ptr(gram), self._ptr(ws), ws.numel(), flags, self._stream()),
                "bkm_gram_weighted_csr_chunk")

    def csr_panel_chunk(self, blk, d, W, out=None, colmax=None, row_offset=0):
        """out = X W over one CSR block ``blk`` of d columns (``W`` float64 (d, l) row-major, ``out`` (n, l) float32 /
        float64 with any row pitch, or None), each element adding its row's entries in column order, and, into
        ``colmax`` (``colmax_new(l)`` records), per column the largest |out_ij| with its lowest global row
        ``row_offset + i`` and its signed value."""
        crow, col, val, n = blk
        l = int(W.shape[1])
        odt = _DT_CODE[out.dtype] if out is not None else _lib.BKM_F64
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_csr_panel_chunk(
                self._ptr(crow), self._ptr(col), self._ptr(val), _DT_CODE[val.dtype], int(n), int(d), int(col.numel()),
                self._ptr(W), l, self._ptr(out), (out.stride(0) if n else l) if out is not None else l, odt,
                self._ptr(colmax), int(row_offset), self._stream()), "bkm_csr_panel_chunk")

    def csc_panel_chunk(self, csc, d, P, out, first=False):
        """out (d, l) (+)= X^T P over the transpose ``csc`` of one block (``P`` float64 (n, l) row-major, ``out`` float64
        (d, l) contiguous), each column's entries added in ascending row order.  ``first`` overwrites."""
        colptr, rows, vals, plan = csc
        nnz = int(rows.numel())
        l = int(out.shape[1])
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_csc_panel_workspace_bytes(int(d), nnz, l, ctypes.byref(nb)),
                   "bkm_csc_panel_workspace_bytes")
        ws = self._scratch("csc_panel", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_csc_panel_chunk(
                self._ptr(colptr), self._ptr(rows), self._ptr(vals), _DT_CODE[vals.dtype], int(d), nnz, self._ptr(plan),
                self._ptr(P), l, self._ptr(out), self._ptr(ws), ws.numel(), flags, self._stream()),
                "bkm_csc_panel_chunk")

    # -- KMeans on sparse CSR blocks ---------------------------------------------------------
    def sparse_pack_centers(self, C64, out=None):
        """The sparse pack of the float64 centres C64 (k, p): one float64 buffer [CT (p, k) | cn (k)] with CT the
        transposed centres and cn their squared norms (``out`` is reused when given)."""
        k, p = C64.shape
        if out is None:
            out = torch.empty(p * k + k, dtype=torch.float64, device=self.device)
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_sparse_pack_workspace_bytes(int(k), int(p), ctypes.byref(nb)),
                   "bkm_sparse_pack_workspace_bytes")
        ws = self._scratch("sparse_pack", nb.value)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_sparse_pack_centers(self._ptr(C64), int(k), int(p), self._ptr(out), self._ptr(ws),
                                                        ws.numel(), self._stream()), "bkm_sparse_pack_centers")
        return out

    def csr_assign_chunk(self, blk, d, pack, k, labels=None, min_dist=None, squared=True, dist_sum=None, counts=None,
                         out=None, mode=0, first=False, loop_state=None):
        """The E-step of one CSR block against a sparse pack: mode 0 writes labels (int32), min_dist (float64, squared
        or not) and adds to dist_sum (1,) / counts (k,) float64 (``first`` overwrites them); modes 1 / 2 write the
        distances / squared distances into ``out`` (n, k) float32 / float64 with any row pitch."""
        crow, col, val, n = blk
        ws = None
        if mode == 0 and (dist_sum is not None or counts is not None):
            nb = ctypes.c_size_t(0)
            _lib.check(self.lib.bkm_csr_assign_workspace_bytes(int(n), int(k), ctypes.byref(nb)),
                       "bkm_csr_assign_workspace_bytes")
            ws = self._scratch("csr_assign", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        odt = _DT_CODE[out.dtype] if out is not None else _lib.BKM_F64
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_csr_assign_chunk(
                self._ptr(crow), self._ptr(col), self._ptr(val), _DT_CODE[val.dtype], int(n), int(d), int(col.numel()),
                self._ptr(pack), int(k), int(mode), self._ptr(labels), self._ptr(min_dist), int(bool(squared)),
                self._ptr(dist_sum), self._ptr(counts), self._ptr(out), (out.stride(0) if n else k) if out is not None
                else k, odt, self._ptr(ws), ws.numel() if ws is not None else 0, flags, self._ptr(loop_state),
                self._stream()), "bkm_csr_assign_chunk")

    def csc_label_sums_chunk(self, csc, d, labels, k, sumsT, first=False, loop_state=None):
        """sumsT (d, k) (+)= X^T onehot(labels) over the transpose ``csc`` of one block, each (column, cluster) sum in
        ascending row order.  ``first`` overwrites."""
        colptr, rows, vals, plan = csc
        nnz = int(rows.numel())
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_csc_label_sums_workspace_bytes(int(d), nnz, int(k), ctypes.byref(nb)),
                   "bkm_csc_label_sums_workspace_bytes")
        ws = self._scratch("csc_label_sums", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_csc_label_sums_chunk(
                self._ptr(colptr), self._ptr(rows), self._ptr(vals), _DT_CODE[vals.dtype], int(d), nnz, self._ptr(plan),
                self._ptr(labels), int(k), self._ptr(sumsT), self._ptr(ws), ws.numel(), flags, self._ptr(loop_state),
                self._stream()), "bkm_csc_label_sums_chunk")

    def sparse_finalize_step(self, red, pack_in, pack_out, state, k, d):
        """bkm_finalize_step on the transposed layout: red = [d*k sumsT | k counts | inertia] -> the shift, the stop
        test and pack_out = the sparse pack of the new centres."""
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_sparse_pack_workspace_bytes(int(k), int(d), ctypes.byref(nb)),
                   "bkm_sparse_pack_workspace_bytes")
        ws = self._scratch("sparse_pack", nb.value)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_sparse_finalize_step(self._ptr(red), self._ptr(pack_in), self._ptr(pack_out),
                                                         self._ptr(state), int(k), int(d), self._ptr(ws), ws.numel(),
                                                         self._stream()), "bkm_sparse_finalize_step")

    def sparse_minibatch_step(self, red, pack_in, w_in, pack_out, w_out, k, d):
        """One mini-batch centre update on the transposed layout (scikit-learn's _minibatch_update_sparse, in float64):
        red = [d*k sumsT | k counts | inertia] of the batch -> pack_out = the sparse pack of the new centres and
        w_out = w_in + counts."""
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_sparse_pack_workspace_bytes(int(k), int(d), ctypes.byref(nb)),
                   "bkm_sparse_pack_workspace_bytes")
        ws = self._scratch("sparse_pack", nb.value)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_sparse_minibatch_step(self._ptr(red), self._ptr(pack_in), self._ptr(w_in),
                                                          self._ptr(pack_out), self._ptr(w_out), int(k), int(d),
                                                          self._ptr(ws), ws.numel(), self._stream()),
                       "bkm_sparse_minibatch_step")

    def csr_kernel_colsum(self, blk, d, pack, l, gamma, colsum, first=False):
        """colsum[j] (+)= sum_i exp(-gamma ||x_i - c_j||^2) over the rows of one CSR block against the sparse pack of the
        l keep rows (float64 [l]); ``first`` overwrites.  The first Nystrom pass of SpectralClustering on sparse X."""
        crow, col, val, n = blk
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_csr_kernel_colsum_workspace_bytes(int(n), int(l), ctypes.byref(nb)),
                   "bkm_csr_kernel_colsum_workspace_bytes")
        ws = self._scratch("csr_kernel_colsum", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_csr_kernel_colsum_chunk(
                self._ptr(crow), self._ptr(col), self._ptr(val), _DT_CODE[val.dtype], int(n), int(d), int(col.numel()),
                self._ptr(pack), int(l), float(gamma), self._ptr(colsum), self._ptr(ws), ws.numel(), flags,
                self._stream()), "bkm_csr_kernel_colsum_chunk")

    def csr_nystrom_embed(self, blk, d, pack, l, gamma, W, out):
        """out[i] = e_i / ||e_i||, e_i = sum_j exp(-gamma (||x_i - c_j||^2 - min_j ||x_i - c_j||^2)) W[j] over one CSR
        block — the second Nystrom pass on sparse X.  ``W`` is (l, k) float64; ``out`` (n, k) float32 / float64 may have
        a padded row pitch."""
        crow, col, val, n = blk
        k = int(W.shape[1])
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_csr_nystrom_embed_chunk(
                self._ptr(crow), self._ptr(col), self._ptr(val), _DT_CODE[val.dtype], int(n), int(d), int(col.numel()),
                self._ptr(pack), int(l), float(gamma), self._ptr(W), k, self._ptr(out), out.stride(0) if n else k,
                _DT_CODE[out.dtype], self.flags, self._stream()), "bkm_csr_nystrom_embed_chunk")

    # -- the SGD family -----------------------------------------------------------------------
    def sgd_block(self, x, order, y, sw, eta, cw, params, w, aw, q, st):
        """One epoch of scikit-learn's ``_plain_sgd`` over the dense block ``x`` (n, d) for P = ``w.shape[0]`` problems:
        ``order`` int32 (P, n), ``y`` float64 (P, n), ``sw`` float64 (n,) or None, ``eta`` float64 (n,) or None
        ('invscaling'), ``cw`` float64 (P, 2), ``params`` an ``_lib.SgdParams``; updates w, aw, q (float64 (P, d)) and
        st (float64 (P, 4): intercept, average intercept, non-finite flag)."""
        n, d = x.shape
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_sgd_block(
                self._ptr(x), int(n), int(d), x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(order),
                self._ptr(y), self._ptr(sw), self._ptr(eta), self._ptr(cw), int(w.shape[0]), ctypes.byref(params),
                self._ptr(w), self._ptr(aw), self._ptr(q), self._ptr(st), self._stream()), "bkm_sgd_block")

    def sgd_csr_block(self, blk, d, order, y, sw, eta, cw, params, w, aw, q, st):
        """``sgd_block`` over one CSR block ``blk`` = (crow, col, val, n) of d columns."""
        crow, col, val, n = blk
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_sgd_csr_block(
                self._ptr(crow), self._ptr(col), self._ptr(val), _DT_CODE[val.dtype], int(n), int(d), int(col.numel()),
                self._ptr(order), self._ptr(y), self._ptr(sw), self._ptr(eta), self._ptr(cw), int(w.shape[0]),
                ctypes.byref(params), self._ptr(w), self._ptr(aw), self._ptr(q), self._ptr(st), self._stream()),
                "bkm_sgd_csr_block")

    def colstats_chunk(self, x, shift, acc, minmax, first=False):
        """The scalers' statistics pass over one chunk, float64 on the device: acc (5, d) (+)= [sum (x - shift) |
        sum (x - shift)^2 over the finite x | NaN count | +inf count | -inf count] and minmax (2, d) = [min | max] over
        the non-NaN x, folded.  ``shift`` float64 (d,) or None; ``first`` overwrites."""
        n, d = x.shape
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_colstats_workspace_bytes(int(n), int(d), ctypes.byref(nb)),
                   "bkm_colstats_workspace_bytes")
        ws = self._scratch("colstats", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_colstats_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(shift), self._ptr(acc),
                self._ptr(minmax), self._ptr(ws), ws.numel(), flags, self._stream()), "bkm_colstats_chunk")

    def radix_state_new(self, d, T):
        """Device state of one radix selection of T order statistics in each of d columns (``radix_select_step``)."""
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_radix_state_bytes(int(d), int(T), ctypes.byref(nb)), "bkm_radix_state_bytes")
        return torch.zeros(int(nb.value), dtype=torch.uint8, device=self.device)

    def radix_hist_chunk(self, x, state, T, rnd, hist, first=False):
        """hist (d, T, 256) float64 (+)= the round-``rnd`` digit counts of the chunk's keys under each target's prefix;
        ``first`` zeroes hist first."""
        n, d = x.shape
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_radix_hist_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(state), int(T), int(rnd),
                self._ptr(hist), flags, self._stream()), "bkm_radix_hist_chunk")

    def radix_select_step(self, hist, state, d, T, rnd, dtype, q):
        """Extend each target's key prefix by the digit that holds its rank (after the round's all-reduce of hist);
        ``q`` the T / 2 quantiles in [0, 1]."""
        qh = (ctypes.c_double * len(q))(*[float(v) for v in q])
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_radix_select_step(self._ptr(hist), self._ptr(state), int(d), int(T), int(rnd),
                                                      _DT_CODE[dtype], ctypes.cast(qh, ctypes.c_void_p),
                                                      self._stream()), "bkm_radix_select_step")

    def quantile_state_new(self, d, n_q):
        """Device state of one selection of the 2 ``n_q`` QuantileTransformer order statistics in each of d columns
        (``quantile_select_step``); column j's record starts at byte j * (16 + 80 n_q)."""
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_quantile_state_bytes(int(d), int(n_q), ctypes.byref(nb)), "bkm_quantile_state_bytes")
        return torch.zeros(int(nb.value), dtype=torch.uint8, device=self.device)

    def quantile_hist_chunk(self, x, state, n_q, rnd, hist, first=False):
        """hist (d, min(2 n_q, 256^rnd), 256) float64 (+)= the round-``rnd`` digit counts of the chunk's keys under each
        live prefix; ``first`` zeroes hist first."""
        n, d = x.shape
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_quantile_hist_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(state), int(n_q), int(rnd),
                self._ptr(hist), flags, self._stream()), "bkm_quantile_hist_chunk")

    def quantile_select_step(self, hist, state, d, n_q, rnd, dtype, qf):
        """Extend each distinct rank's key prefix by one digit and build the next live list (after the round's
        all-reduce of hist); ``qf`` float64 (n_q,) ascending quantiles in [0, 1] on the device."""
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_quantile_select_step(self._ptr(hist), self._ptr(state), int(d), int(n_q), int(rnd),
                                                         _DT_CODE[dtype], self._ptr(qf), self._stream()),
                       "bkm_quantile_select_step")

    def quantile_transform_chunk(self, x, qT, ref, inverse, distribution, clip_lo, clip_hi, out):
        """QuantileTransformer's per-element pass: ``qT`` float64 (d, n_q) quantiles per column, ``ref`` float64
        (n_q,), ``distribution`` 0 uniform / 1 normal; ``out`` float64 (n, d), any row pitch."""
        n, d = x.shape
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_quantile_transform_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(qT), self._ptr(ref),
                int(ref.shape[0]), int(bool(inverse)), int(distribution), float(clip_lo), float(clip_hi),
                self._ptr(out), out.stride(0) if n else d, self._stream()), "bkm_quantile_transform_chunk")

    def impute_stats_chunk(self, x, miss_is_nan, miss, shift, acc, first=False):
        """SimpleImputer's statistics pass over one chunk, float64 on the device: acc (4, d) (+)= [missing count | NaN
        count | inf count | sum (x - shift) over the non-missing finite x].  ``miss`` a value of X's dtype (ignored
        with ``miss_is_nan``); ``shift`` float64 (d,) or None; ``first`` overwrites."""
        n, d = x.shape
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_impute_stats_workspace_bytes(int(n), int(d), ctypes.byref(nb)),
                   "bkm_impute_stats_workspace_bytes")
        ws = self._scratch("impute_stats", nb.value)
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_impute_stats_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], int(bool(miss_is_nan)), float(miss),
                self._ptr(shift), self._ptr(acc), self._ptr(ws), ws.numel(), flags, self._stream()),
                "bkm_impute_stats_chunk")

    def quantile_hist_masked_chunk(self, x, miss, state, n_q, rnd, hist, first=False):
        """``quantile_hist_chunk`` with the elements equal to ``miss`` (a number, not NaN) skipped as well."""
        n, d = x.shape
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_quantile_hist_masked_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], float(miss), self._ptr(state),
                int(n_q), int(rnd), self._ptr(hist), flags, self._stream()), "bkm_quantile_hist_masked_chunk")

    def mode_count_chunk(self, x, miss_is_nan, miss, keys, counts, off, total, first=False):
        """Count the distinct non-missing values of each column of ``x`` (a group of g columns) into the hash tables
        ``keys`` / ``counts`` (uint64 as int64 (total,)), column j owning slots [off[j], off[j + 1]) (``off`` int64
        (g + 1,) on the device); ``first`` resets the tables."""
        n, g = x.shape
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_mode_count_chunk(
                self._ptr(x), n, g, x.stride(0) if n else g, _DT_CODE[x.dtype], int(bool(miss_is_nan)), float(miss),
                self._ptr(keys), self._ptr(counts), self._ptr(off), int(total), flags, self._stream()),
                "bkm_mode_count_chunk")

    def mode_best(self, keys, counts, off, g, total):
        """(best_key int64 (g,) holding uint64 keys, best_count float64 (g,), distinct float64 (g,)) on the device: per
        column the largest count, the smallest key among equal counts (``total`` the tables' slots)."""
        key = torch.empty(g, dtype=torch.int64, device=self.device)
        cnt = torch.empty(g, dtype=torch.float64, device=self.device)
        nd = torch.empty(g, dtype=torch.float64, device=self.device)
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_mode_best_workspace_bytes(int(g), int(total), ctypes.byref(nb)),
                   "bkm_mode_best_workspace_bytes")
        ws = self._scratch("mode_best", nb.value)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_mode_best(self._ptr(keys), self._ptr(counts), self._ptr(off), int(g), int(total),
                                              self._ptr(key), self._ptr(cnt), self._ptr(nd), self._ptr(ws), ws.numel(),
                                              self._stream()), "bkm_mode_best")
        return key, cnt, nd

    def mode_compact(self, keys, counts, off, g, entries):
        """The occupied slots of the tables as rows {column, key >> 32, key & 0xffffffff, count} of ``entries``
        (float64 (m, 4), m at least the number of occupied slots)."""
        cursor = torch.empty(1, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_mode_compact(self._ptr(keys), self._ptr(counts), self._ptr(off), int(g),
                                                 self._ptr(entries), self._ptr(cursor), self._stream()),
                       "bkm_mode_compact")

    def mode_merge(self, entries, keys, counts, off, g, total):
        """Reset the tables and add every row of ``entries`` (float64 (m, 4)) with a non-zero count."""
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_mode_merge(self._ptr(entries), int(entries.shape[0]), self._ptr(keys),
                                               self._ptr(counts), self._ptr(off), int(g), int(total), self._stream()),
                       "bkm_mode_merge")

    def impute_chunk(self, x, miss_is_nan, miss, stats, cols, n_keep, n_ind, n_check, inverse, out, invalid=None):
        """SimpleImputer's fill pass (or its inverse) over one chunk into ``out`` (any row pitch, X's dtype; float32
        for bf16 rows): see include/bkm_b200.h.  ``stats`` float64 (d,), ``cols`` int32 on the device; ``invalid``
        float64 (2,) (+)= the NaN and inf counts of the elements read."""
        n, d = x.shape
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_impute_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], int(bool(miss_is_nan)), float(miss),
                self._ptr(stats), self._ptr(cols), int(n_keep), int(n_ind), int(n_check), int(bool(inverse)),
                self._ptr(out), out.stride(0) if n else int(out.shape[1]), _DT_CODE[out.dtype], self._ptr(invalid),
                self._stream()), "bkm_impute_chunk")

    def distinct_chunk(self, x, keys, counts, off, total, state, first=False):
        """Record the distinct keys of each column of ``x`` (a group of g columns, any element type of
        ``ENCODE_DTYPES``) in the tables ``keys`` / ``counts`` (uint64 as int64 (total,)), column j owning slots
        [off[j], off[j + 1]); ``state`` int64 (2, g) on the device (+)= [occupied slots | status bits: 1 overflow,
        2 holds INT64_MAX]; ``first`` resets tables and state."""
        n, g = x.shape
        flags = self.flags | (_lib.FLAG_FIRST_CHUNK if first else 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_distinct_chunk(
                self._ptr(x), n, g, x.stride(0) if n else g, _ENC_CODE[x.dtype], self._ptr(keys), self._ptr(counts),
                self._ptr(off), int(total), self._ptr(state), flags, self._stream()), "bkm_distinct_chunk")

    def encode_chunk(self, x, cat_keys, cat_off, n_cats, layout, out, unknown, indices=None):
        """One read of ``x`` (n, d): codes, a dense one-hot block or the CSR indices / data of every element, by its
        column's sorted key list (``cat_keys`` int64 holding uint64 keys, ``cat_off`` int64 (d + 1,) on the device).
        ``unknown`` uint64 as int64 (1 + d + d * ENCODE_KEEP,) (+)= the unknown-key counts and kept keys."""
        n, d = x.shape
        if layout == _lib.ENCODE_DENSE:
            ld = int(n_cats)
        else:
            ld = out.stride(0) if layout == _lib.ENCODE_CODES and n else d
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_encode_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _ENC_CODE[x.dtype], self._ptr(cat_keys),
                self._ptr(cat_off), int(n_cats), int(layout), self._ptr(out), ld, _ENC_CODE[out.dtype],
                self._ptr(indices), self._ptr(unknown), self._stream()), "bkm_encode_chunk")

    def decode_chunk(self, codes, cat_vals, cat_off, out, unknown):
        """out (n, d) = cat_vals[cat_off[j] + codes[:, j]] (``codes`` int32 / int64 (n, d), ``cat_vals`` any dtype of
        1, 2, 4 or 8 bytes, ``out`` of the same dtype); codes outside [0, K_j) add to ``unknown``."""
        n, d = codes.shape
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_decode_chunk(
                self._ptr(codes), n, d, codes.stride(0) if n else d, _ENC_CODE[codes.dtype], self._ptr(cat_vals),
                self._ptr(cat_off), cat_vals.element_size(), self._ptr(out), out.stride(0) if n else d,
                self._ptr(unknown), self._stream()), "bkm_decode_chunk")

    def _text_workspace(self, n_bytes, n_docs, n_pairs):
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_text_workspace_bytes(int(n_bytes), int(n_docs), int(n_pairs), ctypes.byref(nb)),
                   "bkm_text_workspace_bytes")
        return self._scratch("text", nb.value)

    def text_tokens_chunk(self, buf, doc_off, min_n, max_n, tok_start, tok_off, pair_off, totals):
        """HashingVectorizer's token pass over the documents packed in ``buf`` (uint8, each document ending in a byte
        that is not a word character, document i at [doc_off[i], doc_off[i + 1])): ``tok_start`` int64 (at least
        len(buf) // 3 + 1,) the tokens' byte positions, ``tok_off`` / ``pair_off`` int64 (n + 1,) each document's first
        token and first n-gram of length in [min_n, max_n]; ``totals`` int64 (3,) [0:2] = the token and n-gram counts."""
        nb, n = int(buf.numel()), int(doc_off.numel()) - 1
        ws = self._text_workspace(nb, n, 0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_text_tokens_chunk(
                self._ptr(buf), nb, self._ptr(doc_off), n, int(min_n), int(max_n), self._ptr(tok_start),
                int(tok_start.numel()), self._ptr(tok_off), self._ptr(pair_off), self._ptr(totals), self._ptr(ws),
                ws.numel(), self._stream()), "bkm_text_tokens_chunk")

    def text_hash_chunk(self, buf, tok_start, tok_off, pair_off, n_tokens, n_pairs, min_n, max_n, lowercase,
                        n_features, alternate_sign, binary, norm, dtype, keys, indptr, scale, totals):
        """Hash every n-gram into ``keys`` (int32 (n_pairs,) holding uint32 2 column + negative sign, sorted per
        document); ``indptr`` int64 (n + 1,) the CSR row offsets and ``scale`` float64 (n,) the row divisors (0: none)
        of the output in ``dtype`` (torch float32 / float64) with ``norm`` None / 'l1' / 'l2'; totals[2] = stored
        entries."""
        nb, n = int(buf.numel()), int(pair_off.numel()) - 1
        ws = self._text_workspace(nb, n, n_pairs)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_text_hash_chunk(
                self._ptr(buf), nb, self._ptr(tok_start), self._ptr(tok_off), self._ptr(pair_off), n, int(n_tokens),
                int(n_pairs), int(min_n), int(max_n), int(bool(lowercase)), int(n_features), int(bool(alternate_sign)),
                int(bool(binary)), _lib.TEXT_NORM[norm], _DT_CODE[dtype], self._ptr(keys), self._ptr(indptr),
                self._ptr(scale), self._ptr(totals), self._ptr(ws), ws.numel(), self._stream()), "bkm_text_hash_chunk")

    def text_write_chunk(self, keys, pair_off, indptr, scale, binary, indices, data):
        """Write the CSR ``indices`` int64 and ``data`` (float32 / float64) of every stored entry."""
        n = int(pair_off.numel()) - 1
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_text_write_chunk(
                self._ptr(keys), self._ptr(pair_off), self._ptr(indptr), self._ptr(scale), n, int(bool(binary)),
                self._ptr(indices), self._ptr(data), _DT_CODE[data.dtype], self._stream()), "bkm_text_write_chunk")

    def affine_chunk(self, x, a, b, op1, op2, out):
        """out = op2(op1(x, a), b) per element (op1: 0 none, 1 subtract a, 2 multiply by a; op2: 0 none, 1 divide by b,
        2 add b), each step rounded once in out's dtype.  ``a``, ``b`` float64 (d,) or None; ``out`` (n, d) float32 /
        float64, any row pitch."""
        n, d = x.shape
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_affine_chunk(
                self._ptr(x), n, d, x.stride(0) if n else d, _DT_CODE[x.dtype], self._ptr(a), self._ptr(b), int(op1),
                int(op2), self._ptr(out), out.stride(0) if n else d, _DT_CODE[out.dtype], self._stream()),
                "bkm_affine_chunk")

    def split_indices_chunk(self, seed, c, start, count, offset):
        """int64 (count,) on the device: ``offset + pi_seed(start + i)``, the split permutation of a block of ``c`` rows
        (include/bkm_b200.h) at positions [start, start + count)."""
        out = torch.empty(int(count), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_split_indices_chunk(int(seed), int(c), int(start), int(count), int(offset),
                                                        self._ptr(out), self._stream()), "bkm_split_indices_chunk")
        return out

    def gather_rows_chunk(self, src, idx, idx_offset=0):
        """``src[idx - idx_offset]`` for a 1-D or 2-D device block of any dtype (rows are copied as bytes; a row pitch
        is honoured, other strides are made contiguous first).  ``idx`` int64 on the device, every value of
        ``idx - idx_offset`` in [0, len(src)): the caller's duty, the kernel does not check."""
        if src.dim() == 2 and src.shape[0] > 1 and (src.stride(1) != 1 or src.stride(0) < src.shape[1]):
            src = src.contiguous()
        elif src.dim() == 1 and src.shape[0] > 1 and src.stride(0) != 1:
            src = src.contiguous()
        idx = idx.contiguous()
        n, count = int(src.shape[0]), int(idx.shape[0])
        out = torch.empty((count,) + tuple(src.shape[1:]), dtype=src.dtype, device=self.device)
        esz = src.element_size()
        row_bytes = esz * (int(src.shape[1]) if src.dim() == 2 else 1)
        if count == 0 or row_bytes == 0:
            return out
        if n == 0:
            raise IndexError("cannot gather rows of an empty block")
        ld_src = src.stride(0) * esz if (src.dim() == 2 and n > 1) else row_bytes
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_gather_rows_chunk(self._ptr(src), n, row_bytes, ld_src, self._ptr(idx),
                                                      int(idx_offset), count, self._ptr(out), row_bytes,
                                                      self._stream()), "bkm_gather_rows_chunk")
        return out

    def metric_chunk(self, a, b, mode, acc, w=None, shift=None, eps=0.0, first=False):
        """One chunk of a scoring reduction (bkm_metric_chunk), float64 on the device.  ``a``, ``b`` contiguous (n,) or
        (n, m) device blocks of any of the types below; ``w`` float64 (n,) or None; ``acc`` float64: METRIC_EQ (2,)
        [sum w [rows equal] | sum w], METRIC_ERR (4, m) [sum (b - a)^2 | sum |b - a| | sum (a - shift) | sum (a - shift)^2]
        with ``shift`` float64 (m,), METRIC_LOGLOSS (2,) [sum -w log q[a] | sum w] with ``a`` int32 class indices and
        ``b`` (n,) or (n, K) probabilities clipped to [eps, 1 - eps] and renormalised.  ``first`` overwrites acc."""
        n = int(b.shape[0])
        m = int(b.shape[1]) if b.dim() == 2 else 1
        nb = ctypes.c_size_t(0)
        _lib.check(self.lib.bkm_metric_workspace_bytes(n, m, int(mode), ctypes.byref(nb)),
                   "bkm_metric_workspace_bytes")
        ws = self._scratch("metric", nb.value)
        flags = _lib.FLAG_FIRST_CHUNK if first else 0
        with torch.cuda.device(self.device):
            _lib.check(self.lib.bkm_metric_chunk(
                self._ptr(a), _METRIC_CODE[a.dtype], self._ptr(b), _METRIC_CODE[b.dtype], self._ptr(w), n, m, int(mode),
                self._ptr(shift), float(eps), self._ptr(acc), self._ptr(ws), ws.numel(), flags, self._stream()),
                "bkm_metric_chunk")

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
