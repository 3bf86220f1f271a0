"""ctypes binding of libb2d (include/b2d.h) — the only way Python reaches the CUDA kernels.

There is deliberately no CPU fallback here: if the shared library cannot be loaded (or built),
importing callers get a ``B2DUnavailableError`` and the GPU strategy refuses to run.
"""
import ctypes
import os
import threading

_LIB = None
_LIB_LOCK = threading.Lock()

HANDLE_BYTES = 256
MAX_WORLD = 8
MAX_BLOCKS = 264

WIRE_FP32, WIRE_BF16 = 0, 1
ALGO_AUTO, ALGO_ONE_SHOT, ALGO_TWO_SHOT, ALGO_NVLS, ALGO_TWO_SHOT_TMA, ALGO_STAGED, ALGO_NVLS_FUSED = 0, 1, 2, 3, 4, 5, 6
PHASE_STAGE, PHASE_EXCHANGE, PHASE_WRITEBACK, PHASE_ALL = 1, 2, 4, 7
FLAG_MEM_LEGACY_IPC, FLAG_MEM_VMM, FLAG_TIMING = 0x0, 0x1, 0x2

WIRE_NAMES = {"fp32": WIRE_FP32, "bf16": WIRE_BF16}
ALGO_NAMES = {"auto": ALGO_AUTO, "one_shot": ALGO_ONE_SHOT, "two_shot": ALGO_TWO_SHOT, "nvls": ALGO_NVLS,
              "two_shot_tma": ALGO_TWO_SHOT_TMA, "staged": ALGO_STAGED, "nvls_fused": ALGO_NVLS_FUSED}

# every symbol include/b2d.h declares (checked by tests/test_cabi.py on a GPU-less box)
EXPORTED_SYMBOLS = [
    "b2d_version", "b2d_ctx_create", "b2d_ctx_export", "b2d_ctx_export_fd", "b2d_handle_set_fd",
    "b2d_ctx_import", "b2d_ctx_finalize", "b2d_mc_supported", "b2d_mc_create", "b2d_mc_join",
    "b2d_mc_bind", "b2d_ctx_destroy", "b2d_last_error", "b2d_ctx_set_timeout", "b2d_ctx_set_max_ctas",
    "b2d_ctx_set_one_shot_max_bytes", "b2d_allreduce_bucket", "b2d_sharded_step", "b2d_reduce_scatter",
    "b2d_allgather", "b2d_barrier", "b2d_arena_alloc", "b2d_arena_reset", "b2d_ctx_stats",
    "b2d_ctx_reset_stats", "b2d_plan", "b2d_ctx_trace", "b2d_ctx_set_tma_ctas",
    "b2d_allreduce_bucket_phased", "b2d_ctx_set_chunk_bytes", "b2d_ctx_set_exch_ctas", "b2d_ctx_set_nvls_auto",
    "b2d_peer_bw", "b2d_pool_bind", "b2d_pool_alloc", "b2d_pool_free", "b2d_ctx_set_inplace",
    "b2d_bucket_register", "b2d_reduce_to_owner", "b2d_adam_push", "b2d_ctx_set_auto_profile",
    "b2d_optim_register", "b2d_bucket_optim", "b2d_bn_register", "b2d_bn_stats_exchange", "b2d_bn_grad_exchange",
    "b2d_adam_push_scaled", "b2d_clip_register", "b2d_clip_norm",
    "b2d_sharded_step64", "b2d_adam_push64", "b2d_adam_push_scaled64", "b2d_bucket_optim64",
]
PROFILE_OVERLAP, PROFILE_LATENCY = 0, 1
RTO_ZERO_GRADS, RTO_ACCUMULATE, RTO_NVLS = 1, 2, 4


class B2DUnavailableError(RuntimeError):
    """libb2d.so is missing and could not be built: the GPU data path cannot run."""


class B2DError(RuntimeError):
    def __init__(self, code, message):
        super().__init__("libb2d error %d: %s" % (code, message))
        self.code = code


class AdamParams(ctypes.Structure):
    """b2d_adam64: the Python floats themselves, so that the library forms torch's constants from the same doubles."""
    _fields_ = [("lr", ctypes.c_double), ("beta1", ctypes.c_double), ("beta2", ctypes.c_double),
                ("eps", ctypes.c_double), ("weight_decay", ctypes.c_double), ("step", ctypes.c_int32),
                ("adamw", ctypes.c_int32), ("zero_grads", ctypes.c_int32), ("pad_", ctypes.c_int32)]


class AdamParams32(ctypes.Structure):
    """b2d_adam: the fp32 form of the C ABI's first Adam entry points."""
    _fields_ = [("lr", ctypes.c_float), ("beta1", ctypes.c_float), ("beta2", ctypes.c_float),
                ("eps", ctypes.c_float), ("weight_decay", ctypes.c_float), ("step", ctypes.c_int32),
                ("adamw", ctypes.c_int32), ("zero_grads", ctypes.c_int32)]


class Seg(ctypes.Structure):
    _fields_ = [("flat_off", ctypes.c_int64), ("len", ctypes.c_int64), ("owner", ctypes.c_int32), ("pad_", ctypes.c_int32)]


class AdamGroup(ctypes.Structure):
    """b2d_adam_group64"""
    _fields_ = [("lo", ctypes.c_int64), ("hi", ctypes.c_int64), ("adam", AdamParams)]


class AdamGroup32(ctypes.Structure):
    """b2d_adam_group"""
    _fields_ = [("lo", ctypes.c_int64), ("hi", ctypes.c_int64), ("adam", AdamParams32), ("pad_", ctypes.c_int32)]


class Stats(ctypes.Structure):
    _fields_ = [("launches", ctypes.c_uint64), ("timed_launches", ctypes.c_uint64),
                ("timed_ms", ctypes.c_double), ("arena_bytes", ctypes.c_uint64),
                ("arena_used", ctypes.c_uint64), ("world", ctypes.c_int32), ("rank", ctypes.c_int32),
                ("device", ctypes.c_int32), ("sm_count", ctypes.c_int32), ("mem_kind", ctypes.c_int32),
                ("mc_bound", ctypes.c_int32), ("last_algo", ctypes.c_int32), ("last_grid", ctypes.c_int32),
                ("last_block", ctypes.c_int32), ("pad_", ctypes.c_int32), ("exch_launches", ctypes.c_uint64),
                ("exch_timed", ctypes.c_uint64), ("exch_ms", ctypes.c_double), ("pool_allocs", ctypes.c_uint64),
                ("pool_digest", ctypes.c_uint64)]

    def as_dict(self):
        return {name: getattr(self, name) for name, _ in self._fields_}


def lib_path():
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libb2d.so")


def _declare(lib):
    c = ctypes
    vp, sz = c.c_void_p, c.c_size_t
    lib.b2d_version.restype = c.c_int
    lib.b2d_last_error.restype = c.c_char_p
    lib.b2d_last_error.argtypes = [vp]
    sigs = {
        "b2d_ctx_create": [c.c_int, c.c_int, c.c_int, sz, c.c_uint, c.POINTER(vp)],
        "b2d_ctx_export": [vp, vp, c.POINTER(sz)],
        "b2d_ctx_export_fd": [vp, c.POINTER(c.c_int)],
        "b2d_handle_set_fd": [vp, sz, c.c_int],
        "b2d_ctx_import": [vp, c.c_int, vp, sz],
        "b2d_ctx_finalize": [vp],
        "b2d_mc_supported": [vp, c.POINTER(c.c_int)],
        "b2d_mc_create": [vp, c.POINTER(c.c_int)],
        "b2d_mc_join": [vp, c.c_int],
        "b2d_mc_bind": [vp],
        "b2d_ctx_destroy": [vp],
        "b2d_ctx_set_timeout": [vp, c.c_uint],
        "b2d_ctx_set_max_ctas": [vp, c.c_int],
        "b2d_ctx_set_tma_ctas": [vp, c.c_int],
        "b2d_ctx_set_one_shot_max_bytes": [vp, sz],
        "b2d_allreduce_bucket": [vp, c.c_int, vp, sz, c.c_int, c.c_float, c.c_int, vp, vp],
        "b2d_allreduce_bucket_phased": [vp, c.c_int, vp, sz, c.c_int, c.c_float, c.c_int, c.c_uint, vp, vp],
        "b2d_ctx_set_chunk_bytes": [vp, sz],
        "b2d_ctx_set_exch_ctas": [vp, c.c_int],
        "b2d_ctx_set_nvls_auto": [vp, c.c_int],
        "b2d_ctx_set_inplace": [vp, c.c_int],
        "b2d_ctx_set_auto_profile": [vp, c.c_int],
        "b2d_optim_register": [vp, c.c_int, c.POINTER(vp), c.POINTER(vp), c.POINTER(vp), c.POINTER(c.c_int64), c.POINTER(c.c_int64), c.c_int],
        "b2d_bucket_optim": [vp, c.c_int, vp, sz, c.c_int, c.POINTER(AdamParams32), c.c_float, vp],
        "b2d_bucket_optim64": [vp, c.c_int, vp, sz, c.c_int, c.POINTER(AdamParams), c.c_float, vp],
        "b2d_peer_bw": [vp, c.c_int, sz, c.c_int, c.c_int, c.POINTER(c.c_double)],
        "b2d_pool_bind": [vp],
        "b2d_bucket_register": [vp, c.c_int, c.POINTER(Seg), c.c_int, c.c_int],
        "b2d_reduce_to_owner": [vp, c.c_int, vp, vp, c.POINTER(c.c_int64), c.c_float, c.c_uint, c.c_uint, vp, vp],
        "b2d_adam_push": [vp, vp, vp, vp, vp, sz, c.POINTER(c.c_int64), c.POINTER(AdamGroup32), c.c_int, c.c_uint, c.c_uint,
                          vp, vp],
        "b2d_adam_push64": [vp, vp, vp, vp, vp, sz, c.POINTER(c.c_int64), c.POINTER(AdamGroup), c.c_int, c.c_uint, c.c_uint,
                            vp, vp],
        "b2d_sharded_step": [vp, c.c_int, vp, vp, vp, vp, sz, c.POINTER(c.c_int64), c.c_int, c.c_float,
                             c.POINTER(AdamParams32), vp, vp],
        "b2d_sharded_step64": [vp, c.c_int, vp, vp, vp, vp, sz, c.POINTER(c.c_int64), c.c_int, c.c_float,
                               c.POINTER(AdamParams), vp, vp],
        "b2d_reduce_scatter": [vp, c.c_int, vp, vp, sz, c.POINTER(c.c_int64), c.c_int, c.c_float, vp, vp],
        "b2d_allgather": [vp, vp, sz, c.POINTER(c.c_int64), vp, vp],
        "b2d_adam_push_scaled": [vp, vp, vp, vp, vp, sz, c.POINTER(c.c_int64), c.POINTER(AdamGroup32), c.c_int, c.c_uint,
                                 c.c_uint, vp, vp, vp],
        "b2d_adam_push_scaled64": [vp, vp, vp, vp, vp, sz, c.POINTER(c.c_int64), c.POINTER(AdamGroup), c.c_int, c.c_uint,
                                   c.c_uint, vp, vp, vp],
        "b2d_clip_register": [vp, c.POINTER(sz)],
        "b2d_clip_norm": [vp, vp, sz, c.c_float, vp, vp, c.c_uint, vp, vp],
        "b2d_bn_register": [vp, c.c_int, c.c_int, c.POINTER(sz)],
        "b2d_bn_stats_exchange": [vp, c.c_int, vp, vp, c.c_float, c.c_float, c.c_float, vp, vp, vp, vp, vp, c.c_uint, vp],
        "b2d_bn_grad_exchange": [vp, c.c_int, vp, vp, vp, vp, c.c_uint, vp],
        "b2d_barrier": [vp, vp],
        "b2d_arena_alloc": [vp, sz, c.POINTER(vp), c.POINTER(sz)],
        "b2d_arena_reset": [vp],
        "b2d_ctx_stats": [vp, c.POINTER(Stats)],
        "b2d_ctx_reset_stats": [vp],
        "b2d_plan": [vp, sz, c.c_int, c.c_int, c.POINTER(c.c_int), c.POINTER(c.c_int), c.POINTER(c.c_int)],
        "b2d_ctx_trace": [vp, c.c_int, c.POINTER(c.c_double), c.POINTER(c.c_int)],
    }
    for name, argtypes in sigs.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = c.c_int
    lib.b2d_pool_alloc.argtypes = [sz, c.c_int, vp]
    lib.b2d_pool_alloc.restype = vp
    lib.b2d_pool_free.argtypes = [vp, sz, c.c_int, vp]
    lib.b2d_pool_free.restype = None


def load(build_if_missing=True):
    """Load (building first if needed and possible) libb2d.so. Raises B2DUnavailableError."""
    global _LIB
    with _LIB_LOCK:
        if _LIB is not None:
            return _LIB
        path = lib_path()
        if build_if_missing:
            try:
                from .csrc.build import build_lib, is_stale, find_nvcc
                if is_stale() and find_nvcc() is not None:
                    build_lib()
            except Exception as e:  # a stale-but-present library is still usable
                if not os.path.exists(path):
                    raise B2DUnavailableError("libb2d.so is missing and building it failed: %s" % e) from e
        if not os.path.exists(path):
            raise B2DUnavailableError(
                "libb2d.so not found at %s; run `python -m ray_lightning_b200.csrc.build` "
                "(there is no CPU fallback for the GPU gradient-sync path)" % path)
        try:
            lib = ctypes.CDLL(path)
        except OSError as e:
            raise B2DUnavailableError("cannot load %s: %s" % (path, e)) from e
        _declare(lib)
        _LIB = lib
        return lib


def _err(lib, ctx, code):
    msg = lib.b2d_last_error(ctx)
    return B2DError(code, msg.decode("utf-8", "replace") if msg else "")


def _stream_ptr(stream):
    """torch.cuda.Stream | int | None -> void* for the C ABI."""
    if stream is None:
        return ctypes.c_void_p(0)
    if isinstance(stream, int):
        return ctypes.c_void_p(stream)
    return ctypes.c_void_p(stream.cuda_stream)


class Context:
    """One rank's libb2d context (thin, exception-raising wrapper over the C ABI)."""

    def __init__(self, rank, world, device, arena_bytes, flags=0):
        self._lib = load()
        self._ctx = ctypes.c_void_p()
        rc = self._lib.b2d_ctx_create(rank, world, device, arena_bytes, flags, ctypes.byref(self._ctx))
        if rc != 0:
            raise _err(self._lib, None, rc)
        self.rank, self.world, self.device, self.flags = rank, world, device, flags

    # -- lifecycle
    def _check(self, rc):
        if rc != 0:
            raise _err(self._lib, self._ctx, rc)

    def export_handle(self):
        buf = ctypes.create_string_buffer(HANDLE_BYTES)
        n = ctypes.c_size_t(HANDLE_BYTES)
        self._check(self._lib.b2d_ctx_export(self._ctx, buf, ctypes.byref(n)))
        return buf.raw[:n.value]

    def export_fd(self):
        fd = ctypes.c_int(-1)
        self._check(self._lib.b2d_ctx_export_fd(self._ctx, ctypes.byref(fd)))
        return fd.value

    def import_handle(self, peer, blob, fd=None):
        buf = ctypes.create_string_buffer(bytes(blob), HANDLE_BYTES)
        if fd is not None:
            rc = self._lib.b2d_handle_set_fd(buf, HANDLE_BYTES, fd)
            if rc != 0:
                raise _err(self._lib, None, rc)
        self._check(self._lib.b2d_ctx_import(self._ctx, peer, buf, HANDLE_BYTES))

    def finalize(self):
        self._check(self._lib.b2d_ctx_finalize(self._ctx))

    def mc_supported(self):
        v = ctypes.c_int(0)
        self._check(self._lib.b2d_mc_supported(self._ctx, ctypes.byref(v)))
        return bool(v.value)

    def mc_create(self):
        fd = ctypes.c_int(-1)
        self._check(self._lib.b2d_mc_create(self._ctx, ctypes.byref(fd)))
        return fd.value

    def mc_join(self, fd):
        self._check(self._lib.b2d_mc_join(self._ctx, fd))

    def mc_bind(self):
        self._check(self._lib.b2d_mc_bind(self._ctx))

    def destroy(self):
        if self._ctx:
            self._lib.b2d_ctx_destroy(self._ctx)
            self._ctx = ctypes.c_void_p()

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass

    # -- knobs
    def set_timeout_ms(self, ms):
        self._check(self._lib.b2d_ctx_set_timeout(self._ctx, int(ms)))

    def set_max_ctas(self, n):
        self._check(self._lib.b2d_ctx_set_max_ctas(self._ctx, int(n)))

    def set_tma_ctas(self, n):
        self._check(self._lib.b2d_ctx_set_tma_ctas(self._ctx, int(n)))

    def set_one_shot_max_bytes(self, n):
        self._check(self._lib.b2d_ctx_set_one_shot_max_bytes(self._ctx, int(n)))

    def set_chunk_bytes(self, n):
        self._check(self._lib.b2d_ctx_set_chunk_bytes(self._ctx, int(n)))

    def set_exch_ctas(self, n):
        self._check(self._lib.b2d_ctx_set_exch_ctas(self._ctx, int(n)))

    def set_nvls_auto(self, enable):
        self._check(self._lib.b2d_ctx_set_nvls_auto(self._ctx, int(bool(enable))))

    def set_auto_profile(self, profile):
        self._check(self._lib.b2d_ctx_set_auto_profile(self._ctx, int(profile)))

    def set_inplace(self, enable):
        self._check(self._lib.b2d_ctx_set_inplace(self._ctx, int(bool(enable))))

    def pool_bind(self, bind=True):
        """Route torch's pluggable-allocator calls (b2d_pool_alloc) to this context's arena, or unbind."""
        self._check(self._lib.b2d_pool_bind(self._ctx if bind else None))

    def peer_bw(self, peer, nbytes, iters=10, mode=1):
        """GB/s this GPU pulls from ``peer``'s arena (mode 0: cudaMemcpyAsync, 1: peer-read kernel)."""
        v = ctypes.c_double(0.0)
        self._check(self._lib.b2d_peer_bw(self._ctx, int(peer), int(nbytes), int(iters), int(mode), ctypes.byref(v)))
        return v.value

    # -- data path (raw pointers; tensor-level wrappers live in comm.py)
    def allreduce_bucket(self, bucket_idx, ptr, n, wire, scale, algo, wait_stream, comm_stream, phases=PHASE_ALL):
        if phases == PHASE_ALL:
            self._check(self._lib.b2d_allreduce_bucket(
                self._ctx, int(bucket_idx), ctypes.c_void_p(ptr), int(n), int(wire), float(scale), int(algo),
                _stream_ptr(wait_stream), _stream_ptr(comm_stream)))
        else:
            self._check(self._lib.b2d_allreduce_bucket_phased(
                self._ctx, int(bucket_idx), ctypes.c_void_p(ptr), int(n), int(wire), float(scale), int(algo),
                int(phases), _stream_ptr(wait_stream), _stream_ptr(comm_stream)))

    def sharded_step(self, slot, grads_ptr, params_ptr, m_ptr, v_ptr, n, shard_off, wire, scale, adam,
                     wait_stream, comm_stream):
        off = (ctypes.c_int64 * len(shard_off))(*[int(x) for x in shard_off])
        self._check(self._lib.b2d_sharded_step64(
            self._ctx, int(slot), ctypes.c_void_p(grads_ptr), ctypes.c_void_p(params_ptr),
            ctypes.c_void_p(m_ptr), ctypes.c_void_p(v_ptr), int(n), off, int(wire), float(scale),
            ctypes.byref(adam), _stream_ptr(wait_stream), _stream_ptr(comm_stream)))

    def reduce_scatter(self, slot, grads_ptr, out_ptr, n, shard_off, wire, scale, wait_stream, comm_stream):
        off = (ctypes.c_int64 * len(shard_off))(*[int(x) for x in shard_off])
        self._check(self._lib.b2d_reduce_scatter(
            self._ctx, int(slot), ctypes.c_void_p(grads_ptr), ctypes.c_void_p(out_ptr), int(n), off,
            int(wire), float(scale), _stream_ptr(wait_stream), _stream_ptr(comm_stream)))

    def allgather(self, buf_ptr, n, shard_off, wait_stream, comm_stream):
        off = (ctypes.c_int64 * len(shard_off))(*[int(x) for x in shard_off])
        self._check(self._lib.b2d_allgather(self._ctx, ctypes.c_void_p(buf_ptr), int(n), off,
                                            _stream_ptr(wait_stream), _stream_ptr(comm_stream)))

    def bucket_register(self, bucket_id, segs, wire):
        """segs: iterable of (flat_off, len, owner)."""
        arr = (Seg * len(segs))(*[Seg(int(o), int(n), int(r), 0) for o, n, r in segs])
        self._check(self._lib.b2d_bucket_register(self._ctx, int(bucket_id), arr, len(segs), int(wire)))

    def reduce_to_owner(self, bucket_id, grads_ptr, reduced_ptr, shard_off, scale, flags, wait_stream, comm_stream, phases=3):
        off = (ctypes.c_int64 * len(shard_off))(*[int(x) for x in shard_off])
        self._check(self._lib.b2d_reduce_to_owner(self._ctx, int(bucket_id), ctypes.c_void_p(grads_ptr),
                                                  ctypes.c_void_p(reduced_ptr), off, float(scale), int(flags), int(phases),
                                                  _stream_ptr(wait_stream), _stream_ptr(comm_stream)))

    def adam_push(self, params_ptr, m_ptr, v_ptr, reduced_ptr, n, shard_off, groups, flags, wait_stream, comm_stream, phases=6,
                  grad_scale_ptr=None):
        """groups: list of (lo, hi, AdamParams) relative to the own shard; empty: push only.  grad_scale_ptr: device fp32
        factor for the gradients (b2d_adam_push_scaled)."""
        off = (ctypes.c_int64 * len(shard_off))(*[int(x) for x in shard_off])
        arr = (AdamGroup * max(len(groups), 1))(*[AdamGroup(int(lo), int(hi), a) for lo, hi, a in groups])
        args = (self._ctx, ctypes.c_void_p(params_ptr), ctypes.c_void_p(m_ptr or 0), ctypes.c_void_p(v_ptr or 0),
                ctypes.c_void_p(reduced_ptr or 0), int(n), off, arr, len(groups), int(flags), int(phases),
                _stream_ptr(wait_stream), _stream_ptr(comm_stream))
        if grad_scale_ptr is None:
            self._check(self._lib.b2d_adam_push64(*args))
        else:
            self._check(self._lib.b2d_adam_push_scaled64(*args, ctypes.c_void_p(grad_scale_ptr)))

    def clip_register(self):
        """Returns the arena offset of the clip exchange's region."""
        off = ctypes.c_size_t()
        self._check(self._lib.b2d_clip_register(self._ctx, ctypes.byref(off)))
        return off.value

    def clip_norm(self, x_ptr, n, max_norm, norm_ptr, coef_ptr, phases, wait_stream, comm_stream):
        vp = ctypes.c_void_p
        self._check(self._lib.b2d_clip_norm(self._ctx, vp(x_ptr), int(n), float(max_norm), vp(norm_ptr), vp(coef_ptr),
                                            int(phases), _stream_ptr(wait_stream), _stream_ptr(comm_stream)))

    def optim_register(self, bucket_id, param_ptrs, state1_ptrs, state2_ptrs, bucket_offs, numels):
        n = len(param_ptrs)
        arr = lambda ps: (ctypes.c_void_p * n)(*[int(p) for p in ps]) if ps is not None else None
        self._check(self._lib.b2d_optim_register(
            self._ctx, int(bucket_id), arr(param_ptrs), arr(state1_ptrs), arr(state2_ptrs),
            (ctypes.c_int64 * n)(*[int(o) for o in bucket_offs]), (ctypes.c_int64 * n)(*[int(x) for x in numels]), n))

    def bucket_optim(self, bucket_id, grads_ptr, n, kind, hp, momentum, stream):
        self._check(self._lib.b2d_bucket_optim64(self._ctx, int(bucket_id), ctypes.c_void_p(grads_ptr), int(n), int(kind),
                                               ctypes.byref(hp), float(momentum), _stream_ptr(stream)))

    def bn_register(self, layer_id, channels):
        """Returns the arena offset of the layer's exchange region."""
        off = ctypes.c_size_t()
        self._check(self._lib.b2d_bn_register(self._ctx, int(layer_id), int(channels), ctypes.byref(off)))
        return off.value

    def bn_stats_exchange(self, layer_id, mean_ptr, invstd_ptr, count, eps, momentum, mean_out_ptr, invstd_out_ptr,
                          counts_out_ptr, running_mean_ptr, running_var_ptr, phases, stream):
        vp = ctypes.c_void_p
        self._check(self._lib.b2d_bn_stats_exchange(
            self._ctx, int(layer_id), vp(mean_ptr), vp(invstd_ptr), float(count), float(eps), float(momentum),
            vp(mean_out_ptr), vp(invstd_out_ptr), vp(counts_out_ptr), vp(running_mean_ptr), vp(running_var_ptr),
            int(phases), _stream_ptr(stream)))

    def bn_grad_exchange(self, layer_id, sum_dy_ptr, sum_dy_xmu_ptr, sum_dy_out_ptr, sum_dy_xmu_out_ptr, phases, stream):
        vp = ctypes.c_void_p
        self._check(self._lib.b2d_bn_grad_exchange(self._ctx, int(layer_id), vp(sum_dy_ptr), vp(sum_dy_xmu_ptr),
                                                   vp(sum_dy_out_ptr), vp(sum_dy_xmu_out_ptr), int(phases),
                                                   _stream_ptr(stream)))

    def barrier(self, stream):
        self._check(self._lib.b2d_barrier(self._ctx, _stream_ptr(stream)))

    def arena_alloc(self, nbytes):
        p, off = ctypes.c_void_p(), ctypes.c_size_t()
        self._check(self._lib.b2d_arena_alloc(self._ctx, int(nbytes), ctypes.byref(p), ctypes.byref(off)))
        return p.value, off.value

    def arena_reset(self):
        self._check(self._lib.b2d_arena_reset(self._ctx))

    def stats(self):
        s = Stats()
        self._check(self._lib.b2d_ctx_stats(self._ctx, ctypes.byref(s)))
        return s.as_dict()

    def reset_stats(self):
        self._check(self._lib.b2d_ctx_reset_stats(self._ctx))

    def trace(self, enable=True, read=False):
        """Debug: enable phase stamping / read the last launch's per-phase microseconds."""
        if not read:
            self._check(self._lib.b2d_ctx_trace(self._ctx, int(enable), None, None))
            return None
        buf = (ctypes.c_double * 8)()
        n = ctypes.c_int(0)
        self._check(self._lib.b2d_ctx_trace(self._ctx, int(enable), buf, ctypes.byref(n)))
        return [buf[i] for i in range(n.value)]

    def plan(self, n, wire, algo=ALGO_AUTO):
        a, g, b = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        self._check(self._lib.b2d_plan(self._ctx, int(n), int(wire), int(algo), ctypes.byref(a),
                                       ctypes.byref(g), ctypes.byref(b)))
        return a.value, g.value, b.value
