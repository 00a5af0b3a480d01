"""ctypes binding of the C ABI in ``include/emcee_b200.h``.

The shared library ``libemcee_b200.so`` is built in-tree by
``__graft_entry__.build()`` (or ``make -C emcee_b200/csrc``).  There is no
fallback: if the library is missing, or no CUDA device is visible when an
engine is created, the caller gets an exception.
"""

import ctypes as C
import os

import numpy as np

__all__ = ["lib", "Engine", "Chain", "EngineError", "device_count", "LIB_PATH", "EbMove", "DeviceRows", "DeviceArray"]

HERE = os.path.dirname(os.path.abspath(__file__))
# EMCEE_B200_LIB: developer override (A/B of two builds); the product always loads the in-tree library
LIB_PATH = os.environ.get("EMCEE_B200_LIB") or os.path.join(HERE, "libemcee_b200.so")

EB_OK = 0
EB_ERR_INVALID = -1
EB_ERR_CUDA = -2
EB_ERR_COMM = -3
EB_ERR_STATE = -4
EB_ERR_UNSUPPORTED = -5
EB_ERR_NOMEM = -6
EB_ERR_CALLBACK = -7
EB_ERR_NAN_LOGPROB = -10
EB_ERR_INF_PARAM = -11
EB_ERR_NAN_PARAM = -12
EB_ERR_FEW_WALKERS = -13
EB_ERR_NAN_INITIAL = -14
EB_ERR_SINGULAR = -15

EB_COMM_ID_BYTES = 128
EB_IPC_BLOB_BYTES = 256
EB_COMM_ALLGATHER = 0
EB_COMM_P2P = 1
EB_CALLBACK_HOST = 0
EB_CHAIN_COORDS = 0
EB_CHAIN_LOG_PROB = 1
EB_CALLBACK_DEVICE = 1
EB_CALLBACK_GRAPH = 2
EB_MAX_PROPOSAL_SLOTS = 64  # user proposals one engine can hold (eb_move_set_proposal)
EB_DRAW_KINDS = {"uniform": 0, "normal": 1}  # eb_move_set_proposal_graphs: EB_DRAW_UNIFORM, EB_DRAW_NORMAL
EB_MAX_GRAPH_DRAWS = 2**19  # draws per row of a captured proposal: the counter's 18-bit sub-index holds k < 2**18
EB_STREAM_UNKNOWN = 2**64 - 1  # eb_callback_result: the producer named no stream -> wait for the whole device

MODEL_KINDS = {"gauss_iso": 0, "gauss_dense": 1, "rosenbrock": 2, "ring": 3}
MOVE_KINDS = {"stretch": 0, "de": 1, "snooker": 2, "walk": 3, "gaussian": 4, "user": 5, "user_mh": 6, "kde": 7}


class EbMove(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("nsplits", C.c_int32),
        ("randomize_split", C.c_int32),
        ("live_dangerously", C.c_int32),
        ("weight", C.c_double),
        ("p0", C.c_double),
        ("p1", C.c_double),
        # ABI 2: GaussianMove
        ("mode", C.c_int32),
        ("reserved", C.c_int32),
        ("seq_index", C.c_int64),
        ("cov", C.POINTER(C.c_double)),
        ("ncov", C.c_uint64),
    ]


class EbGraph(C.Structure):
    _fields_ = [
        ("m", C.c_int64),
        ("exec", C.c_uint64),
        ("x", C.c_void_p),
        ("x_row_stride_bytes", C.c_int64),
        ("lp", C.c_void_p),
        ("lp_stride_bytes", C.c_int64),
    ]


class EbProposalGraph(C.Structure):
    _fields_ = [
        ("split", C.c_int32),
        ("ns", C.c_int64),
        ("exec", C.c_uint64),
        ("s", C.c_void_p),
        ("s_row_stride_bytes", C.c_int64),
        ("c", C.c_void_p),
        ("c_row_stride_bytes", C.c_int64),
        ("draws", C.c_void_p),
        ("draws_row_stride_bytes", C.c_int64),
        ("q", C.c_void_p),
        ("q_row_stride_bytes", C.c_int64),
        ("factors", C.c_void_p),
        ("factors_stride_bytes", C.c_int64),
    ]


class EngineError(RuntimeError):
    """A failing C-ABI call that does not map onto one of the reference's own
    exception types."""


_dp = C.POINTER(C.c_double)
# eb_logprob_fn: (user, x, m, ndim, lp, stream) -> 0 | non-zero
LOGPROB_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, _dp, C.c_int64, C.c_int64, _dp, C.c_void_p)
# eb_proposal_fn: (user, step, split, s, ns, c, c_counts, nsets, ndim, q, factors, stream) -> 0 | non-zero
PROPOSAL_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.c_int32, _dp, C.c_int64, _dp, C.POINTER(C.c_int64),
                          C.c_int32, C.c_int64, _dp, _dp, C.c_void_p)
_SIGNATURES = {
    "eb_abi_version": (C.c_int, []),
    "eb_device_count": (C.c_int, []),
    "eb_create": (C.c_int, [C.c_int, C.c_int64, C.c_int64, C.c_uint64, C.POINTER(C.c_void_p)]),
    "eb_create_batch": (C.c_int, [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_uint64),
                                  C.POINTER(C.c_void_p)]),
    "eb_batch_rng_get": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "eb_batch_rng_set": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint64]),
    "eb_destroy": (C.c_int, [C.c_void_p]),
    "eb_last_error": (C.c_char_p, [C.c_void_p]),
    "eb_model_set": (C.c_int, [C.c_void_p, C.c_int, _dp, C.c_size_t]),
    "eb_model_set_bounds": (C.c_int, [C.c_void_p, _dp, _dp]),
    "eb_model_set_callback": (C.c_int, [C.c_void_p, LOGPROB_FN, C.c_void_p, C.c_int]),
    "eb_model_set_graphs": (C.c_int, [C.c_void_p, C.POINTER(EbGraph), C.c_size_t]),
    "eb_callback_result": (C.c_int, [C.c_void_p, _dp, C.c_void_p, C.c_int64, C.c_int64, C.c_uint64]),
    "eb_callback_blobs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_uint64]),
    "eb_move_set_proposal": (C.c_int, [C.c_void_p, C.c_int32, PROPOSAL_FN, C.c_void_p, C.c_int]),
    "eb_move_set_proposal_graphs": (C.c_int, [C.c_void_p, C.c_int32, C.c_int, C.c_int64, C.POINTER(EbProposalGraph),
                                              C.c_size_t]),
    "eb_proposal_result": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_uint64]),
    "eb_set_state": (C.c_int, [C.c_void_p, _dp, _dp]),
    "eb_get_state": (C.c_int, [C.c_void_p, _dp, _dp]),
    "eb_set_state_blobs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "eb_get_blobs": (C.c_int, [C.c_void_p, C.c_void_p]),
    "eb_compute_log_prob_blobs": (
        C.c_int, [C.c_void_p, _dp, C.c_size_t, _dp, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)],
    ),
    "eb_owned_rows": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "eb_get_state_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _dp, _dp]),
    "eb_compute_log_prob": (C.c_int, [C.c_void_p, _dp, C.c_size_t, _dp]),
    "eb_set_rng": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64]),
    "eb_get_rng": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "eb_step": (C.c_int, [C.c_void_p, C.POINTER(EbMove), C.c_size_t, C.c_uint64, C.POINTER(C.c_uint8)]),
    "eb_step_store": (
        C.c_int,
        [C.c_void_p, C.POINTER(EbMove), C.c_size_t, C.c_uint64, C.c_uint64, _dp, _dp, _dp],
    ),
    "eb_step_store_blobs": (
        C.c_int,
        [C.c_void_p, C.POINTER(EbMove), C.c_size_t, C.c_uint64, C.c_uint64, _dp, _dp, _dp, C.c_void_p],
    ),
    "eb_step_store_chain": (
        C.c_int,
        [C.c_void_p, C.POINTER(EbMove), C.c_size_t, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64],
    ),
    "eb_chain_create": (C.c_int, [C.c_int, C.c_int64, C.c_int64, C.POINTER(C.c_void_p)]),
    "eb_chain_destroy": (C.c_int, [C.c_void_p]),
    "eb_chain_last_error": (C.c_char_p, [C.c_void_p]),
    "eb_chain_grow": (C.c_int, [C.c_void_p, C.c_uint64]),
    "eb_chain_capacity": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "eb_chain_write": (C.c_int, [C.c_void_p, C.c_uint64, _dp, _dp, C.POINTER(C.c_uint8)]),
    "eb_chain_read": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, _dp, _dp]),
    "eb_chain_accepted": (C.c_int, [C.c_void_p, _dp]),
    "eb_chain_autocorr": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, _dp]),
    "eb_chain_select": (
        C.c_int,
        [C.c_void_p, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), C.c_size_t, _dp,
         C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)],
    ),
    "eb_chain_moments": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, _dp, _dp, C.POINTER(C.c_uint64)]),
    "eb_chain_histogram": (
        C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, _dp, _dp, C.POINTER(C.c_uint64)],
    ),
    "eb_chain_histogram2d": (
        C.c_int,
        [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32), C.c_size_t, C.c_uint32, _dp,
         C.POINTER(C.c_uint64)],
    ),
    "eb_get_naccepted": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "eb_reset_counters": (C.c_int, [C.c_void_p]),
    "eb_move_picks": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_size_t]),
    "eb_moments": (C.c_int, [C.c_void_p, _dp, _dp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "eb_histograms_config": (
        C.c_int,
        [C.c_void_p, C.c_uint64, C.c_uint32, _dp, _dp, C.c_int, C.POINTER(C.c_uint32), C.c_size_t, C.c_uint32, _dp],
    ),
    "eb_histograms": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "eb_trace_config": (C.c_int, [C.c_void_p, C.c_uint64]),
    "eb_trace_count": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "eb_trace_read": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), _dp]),
    "eb_trace_best": (C.c_int, [C.c_void_p, _dp, _dp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "eb_reservoir_config": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64]),
    "eb_reservoir_count": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "eb_reservoir_read": (C.c_int, [C.c_void_p, _dp, _dp, C.POINTER(C.c_uint64), C.POINTER(C.c_int64)]),
    "eb_reservoir_read_to": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64),
                                       C.POINTER(C.c_int64)]),
    "eb_running_acf_config": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64]),
    "eb_running_acf_count": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "eb_running_acf_read": (C.c_int, [C.c_void_p, _dp]),
    "eb_window_config": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64]),
    "eb_window_count": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "eb_window_steps": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "eb_window_chain": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "eb_walkers_gram": (C.c_int, [C.c_void_p, _dp, C.c_size_t, _dp, C.POINTER(C.c_int)]),
    "eb_autocorr": (C.c_int, [C.c_void_p, _dp, C.c_size_t, C.c_size_t, C.c_size_t, _dp]),
    "eb_last_step_timing": (C.c_int, [C.c_void_p, _dp, C.POINTER(C.c_uint64)]),
    "eb_debug_taps": (
        C.c_int,
        [C.c_void_p, C.POINTER(C.c_int64), _dp, _dp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)],
    ),
    "eb_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64]),
    "eb_debug_timeline": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.c_size_t, C.POINTER(C.c_size_t)]),
    "eb_last_kernel_name": (C.c_char_p, [C.c_void_p]),
    "eb_last_kernel_variant": (C.c_char_p, [C.c_void_p]),
    "eb_microbench": (C.c_int, [C.c_int, C.c_int, _dp]),
    "eb_host_alloc": (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p)]),
    "eb_host_free": (C.c_int, [C.c_void_p]),
    "eb_comm_id": (C.c_int, [C.c_char_p]),
    "eb_comm_init": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int]),
    "eb_comm_export": (C.c_int, [C.c_void_p, C.c_char_p]),
    "eb_comm_import": (C.c_int, [C.c_void_p, C.c_char_p]),
    "eb_comm_probe": (C.c_int, [C.c_void_p, C.c_int, C.c_int, _dp]),
    "eb_device_alloc": (C.c_int, [C.c_int, C.c_size_t, C.POINTER(C.c_void_p)]),
    "eb_device_free": (C.c_int, [C.c_int, C.c_void_p]),
    "eb_device_copy": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_uint64]),
    "eb_set_state_from": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_uint64]),
    "eb_get_state_to": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "eb_compute_log_prob_from": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_uint64]),
    "eb_chain_read_to": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]),
    "eb_chain_read_segments_to": (
        C.c_int, [C.c_void_p, C.c_int64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]),
    "eb_chain_autocorr_segments": (C.c_int, [C.c_void_p, C.c_int64, C.c_uint64, C.c_uint64, C.c_uint64, _dp]),
    "eb_chain_select_segments": (
        C.c_int,
        [C.c_void_p, C.c_int64, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), C.c_size_t, _dp,
         C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)],
    ),
    "eb_chain_moments_segments": (
        C.c_int, [C.c_void_p, C.c_int64, C.c_uint64, C.c_uint64, C.c_uint64, _dp, _dp, C.POINTER(C.c_uint64)]),
    "eb_chain_histogram_segments": (
        C.c_int,
        [C.c_void_p, C.c_int64, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, _dp, _dp,
         C.POINTER(C.c_uint64)],
    ),
    "eb_chain_histogram2d_segments": (
        C.c_int,
        [C.c_void_p, C.c_int64, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32), C.c_size_t, C.c_uint32,
         _dp, C.POINTER(C.c_uint64)],
    ),
}

_lib = None


def lib():
    """The loaded shared library (loaded once; raises if it was not built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "emcee_b200: %s is missing -- build it with `python -c 'import "
                "__graft_entry__ as g; g.build()'` or `make -C emcee_b200/csrc`. "
                "There is no CPU fallback." % LIB_PATH
            )
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            if os.environ.get("EMCEE_B200_LIB") and not hasattr(handle, name):
                continue  # A/B against an older build
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def exported_symbols():
    return sorted(_SIGNATURES)


def device_count():
    return int(lib().eb_device_count())


def microbench(what, warps_per_sm=16):
    """TFLOP/s (what = 0 DFMA, 1..3 DMMA shapes) or GB/s (4 = HBM copy)."""
    out = C.c_double()
    rc = lib().eb_microbench(int(what), int(warps_per_sm), C.byref(out))
    if rc != EB_OK:
        raise EngineError("eb_microbench failed (%d)" % rc)
    return float(out.value)


class _PinnedOwner(object):
    def __init__(self, ptr):
        self.ptr = ptr

    def __del__(self):
        try:
            lib().eb_host_free(self.ptr)
        except Exception:
            pass


def pinned_empty(shape, dtype=np.float64):
    """numpy array in page-locked host memory (full-speed H2D / D2H)."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    ptr = C.c_void_p()
    rc = lib().eb_host_alloc(max(n, 1), C.byref(ptr))
    if rc != EB_OK:
        raise EngineError("eb_host_alloc(%d) failed" % n)
    buf = (C.c_char * max(n, 1)).from_address(ptr.value)
    buf._owner = _PinnedOwner(ptr)  # freed when the last array viewing `buf` dies
    return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)


def _as_dp(a):
    return a.ctypes.data_as(_dp)


def _f64(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if shape is not None and a.shape != shape:
        raise ValueError("incompatible input dimensions {0}".format(a.shape))
    return a


def _raise(rc, msg):
    if rc in (EB_ERR_INVALID, EB_ERR_NAN_LOGPROB, EB_ERR_INF_PARAM, EB_ERR_NAN_PARAM, EB_ERR_NAN_INITIAL):
        raise ValueError(msg)
    if rc == EB_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    if rc == EB_ERR_FEW_WALKERS:
        raise RuntimeError(msg)
    if rc == EB_ERR_NOMEM:
        raise MemoryError(msg)
    if rc == EB_ERR_SINGULAR:
        raise np.linalg.LinAlgError(msg)
    raise EngineError("%s (eb_status %d)" % (msg, rc))


def _raise_no_ctx(rc):
    """The error of a failing call without a context (``eb_device_alloc``, ...): its message is eb_last_error(NULL)."""
    _raise(rc, lib().eb_last_error(None).decode())


class DeviceArray(object):
    """A C-contiguous float64 array in device memory owned by the package: what ``cuda_results=True`` states and the
    ``cuda=True`` reads of a ``DeviceBackend`` return.

    It exposes the CUDA Array Interface (v3) with ``stream: None``: the data is complete when the array is handed
    out, so a consumer needs no synchronisation.  ``torch.as_tensor(a, device="cuda")`` and ``cupy.asarray(a)``
    wrap it without a copy and keep it alive; the memory is freed when the last reference goes.  ``get()``
    returns a numpy copy.  A zero-size array has data pointer 0.  Pickling goes through the host."""

    __slots__ = ("_ptr", "_shape", "_device")

    def __init__(self, shape, device=0):
        self._ptr = 0
        self._shape = tuple(int(n) for n in shape)
        self._device = int(device)
        ptr = C.c_void_p()
        rc = lib().eb_device_alloc(self._device, self.nbytes, C.byref(ptr))
        if rc != EB_OK:
            _raise_no_ctx(rc)
        self._ptr = ptr.value or 0

    def __del__(self):
        if self._ptr:
            try:
                lib().eb_device_free(self._device, C.c_void_p(self._ptr))
            except Exception:
                pass
            self._ptr = 0

    @property
    def __cuda_array_interface__(self):
        return {"shape": self._shape, "typestr": "<f8", "data": (self._ptr, False), "strides": None, "version": 3,
                "stream": None}

    @property
    def shape(self):
        return self._shape

    @property
    def dtype(self):
        return np.dtype(np.float64)

    @property
    def device(self):
        """The CUDA device ordinal the memory lives on."""
        return self._device

    @property
    def ndim(self):
        return len(self._shape)

    @property
    def size(self):
        return int(np.prod(self._shape, dtype=np.int64))

    @property
    def nbytes(self):
        return 8 * self.size

    def __len__(self):
        if not self._shape:
            raise TypeError("len() of a 0-d DeviceArray")
        return self._shape[0]

    def _copy_from(self, src, stream=0):
        if self.nbytes:
            rc = lib().eb_device_copy(self._device, C.c_void_p(self._ptr), C.c_void_p(src), self.nbytes, self.nbytes,
                                      1, int(stream))
            if rc != EB_OK:
                _raise_no_ctx(rc)

    def get(self):
        """A numpy copy of the array."""
        out = np.empty(self._shape, dtype=np.float64)
        if self.nbytes:
            rc = lib().eb_device_copy(self._device, C.c_void_p(out.ctypes.data), C.c_void_p(self._ptr), self.nbytes,
                                      self.nbytes, 1, 0)
            if rc != EB_OK:
                _raise_no_ctx(rc)
        return out

    def copy(self):
        """A new DeviceArray with the same values (a device-to-device copy)."""
        out = DeviceArray(self._shape, self._device)
        out._copy_from(self._ptr)
        return out

    def __deepcopy__(self, memo):
        return self.copy()

    def __reduce__(self):
        return _device_array_from_host, (self.get(), self._device)

    def __repr__(self):
        return "DeviceArray(shape=%s, dtype=float64, device=%d)" % (self._shape, self._device)


def _device_array_from_host(a, device):
    """Unpickling: upload a host array into a new :class:`DeviceArray`."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    out = DeviceArray(a.shape, device)
    out._copy_from(a.ctypes.data)
    return out


def is_cuda_array(obj):
    """Whether ``obj`` exposes the CUDA Array Interface (a torch / CuPy / Numba device array, a :class:`DeviceArray`)."""
    return obj is not None and hasattr(obj, "__cuda_array_interface__")


def cuda_array_device(obj):
    """The CUDA device ordinal an array object names -- ``DeviceArray.device``, a torch ``device.index``, a CuPy
    ``device.id`` -- or None when it names none (the engine then checks the pointer itself)."""
    dev = getattr(obj, "device", None)
    if isinstance(dev, (int, np.integer)) and not isinstance(dev, bool):
        return int(dev)
    if getattr(dev, "type", None) == "cuda" and getattr(dev, "index", None) is not None:
        return int(dev.index)
    if isinstance(getattr(dev, "id", None), int):
        return int(dev.id)
    return None


class CudaRows(object):
    """A validated CUDA array for the device-memory transfers: its data pointer, first-axis stride in bytes and
    the stream its producer names (the ``eb_callback_result`` encoding)."""

    __slots__ = ("ptr", "stride", "stream", "shape")

    def __init__(self, obj, shape, device, what):
        cai = obj.__cuda_array_interface__
        got = tuple(int(n) for n in cai["shape"])
        if got != tuple(shape):
            raise ValueError("incompatible input dimensions {0}".format(got))
        if np.dtype(cai["typestr"]) != np.float64:
            raise TypeError("%s must be a float64 CUDA array, got %s" % (what, np.dtype(cai["typestr"])))
        if cai.get("mask") is not None:
            raise ValueError("masked CUDA arrays are not supported as %s" % what)
        dev = cuda_array_device(obj)
        if dev is not None and dev != int(device):
            raise ValueError("%s is on CUDA device %d; the sampler runs on device %d" % (what, dev, int(device)))
        row = 8 * int(np.prod(got[1:], dtype=np.int64))
        stride = row
        strides = cai.get("strides")
        if strides is not None:
            strides = tuple(int(n) for n in strides)
            if any(n > 1 and st != 8 for n, st in zip(got[1:], strides[1:])):
                raise ValueError("the rows of %s must be contiguous; only the first axis may be strided" % what)
            if got[0] > 1:
                stride = strides[0]
                if stride < row or stride % 8:
                    raise ValueError("the first-axis stride of %s (%d bytes) must be a multiple of 8 bytes and at "
                                     "least a row (%d bytes)" % (what, stride, row))
        self.ptr = int(cai["data"][0] or 0)
        self.stride = stride
        # a "stream" entry is the producer's word on ordering (None: none needed); without one (interface v2, which
        # torch exports) the data may still be in flight on any stream, so the engine waits for all of them
        self.stream = (cai["stream"] or 0) if "stream" in cai else EB_STREAM_UNKNOWN
        self.shape = got

    def download(self, device):
        """A numpy copy of the rows, ordered after the producer's stream (``eb_device_copy``)."""
        out = np.empty(self.shape, dtype=np.float64)
        width = out.itemsize * int(np.prod(self.shape[1:], dtype=np.int64))
        if out.size:
            rc = lib().eb_device_copy(int(device), C.c_void_p(out.ctypes.data), C.c_void_p(self.ptr), width,
                                      self.stride, self.shape[0], int(self.stream))
            if rc != EB_OK:
                _raise_no_ctx(rc)
        return out


def _one_stream(*streams):
    """The stream one copy of several producers' arrays waits for: the one they name, or the whole device."""
    named = set(streams) - {0}
    return named.pop() if len(named) == 1 else (EB_STREAM_UNKNOWN if named else 0)


class DeviceRows(object):
    """The ``[m, ndim]`` float64 rows a device-mode callback receives: an immutable object with the
    CUDA Array Interface (v3) whose ``stream`` is the engine's stream; the rows are complete when the
    function is called, so a consumer that ignores ``stream`` reads them correctly too.  The memory is a scratch copy of the proposals that belongs to the engine: the function may
    overwrite it (so the interface's read-only flag is False, which torch requires), and it is valid
    only during the call; afterwards the interface raises ``RuntimeError``."""

    __slots__ = ("_cai",)
    _what = "a log-probability callback"

    def __init__(self, ptr, m, ndim, stream):
        self._cai = {"shape": (int(m), int(ndim)), "typestr": "<f8", "data": (int(ptr or 0), False),
                     "strides": None, "version": 3, "stream": int(stream) if stream else None}

    @property
    def __cuda_array_interface__(self):
        if self._cai is None:
            raise RuntimeError("the rows of %s are only valid during the call" % self._what)
        return dict(self._cai)

    @property
    def shape(self):
        return self.__cuda_array_interface__["shape"]

    def _release(self):
        self._cai = None


class ProposalRows(DeviceRows):
    """The rows a device-mode user proposal receives (``s``, each ``c[j]``, or the ensemble): as
    :class:`DeviceRows`, engine scratch valid only during the call."""

    __slots__ = ()
    _what = "a user proposal"


def _proposal_arrays(out):
    """``(q, factors)`` of a proposal's result, or the error for anything else."""
    try:
        q, f = out
    except (TypeError, ValueError):
        raise ValueError("the proposal must return (q, factors)") from None
    return q, f


def _check_proposal(shape, dtype, want, what):
    if tuple(shape) != want:
        raise ValueError("the proposal returned %s of shape %s; expected %s" % (what, tuple(shape), want))
    if np.dtype(dtype) != np.float64:
        raise TypeError("the proposal must return float64 %s, got %s" % (what, np.dtype(dtype)))


def make_proposal_trampoline(h, propose, setup, where, failure, seed_box):
    """The C proposal function of one schedule entry: calls ``propose(s, c, random)`` (host mode: fresh ndarrays the
    function owns; device mode: :class:`ProposalRows`) and hands ``(q, factors)`` to the engine; ``setup(coords)``
    for the setup call (split -1).  ``random`` = ``moves.user_random(seed_box[0], step, split)``.  Any exception is
    stored as ``failure[0]`` and the engine is told to stop (``EB_ERR_CALLBACK``)."""
    from .moves.user import user_random

    def host(user, step, split, s, ns, c, counts, nsets, ndim, q, f):
        S = np.ctypeslib.as_array(s, shape=(ns, ndim)).copy()
        if split < 0:
            setup(S)
            return
        sizes = [int(counts[j]) for j in range(nsets)]
        cs = []
        if nsets:
            allc = np.ctypeslib.as_array(c, shape=(sum(sizes), ndim))
            cs = [a.copy() for a in np.split(allc, np.cumsum(sizes)[:-1])]
        qo, fo = _proposal_arrays(propose(S, cs, user_random(seed_box[0], step, split)))
        qa, fa = np.asarray(qo), np.asarray(fo)
        _check_proposal(qa.shape, qa.dtype, (ns, ndim), "q")
        _check_proposal(fa.shape, fa.dtype, (ns,), "factors")
        np.ctypeslib.as_array(q, shape=(ns, ndim))[:] = qa
        np.ctypeslib.as_array(f, shape=(ns,))[:] = fa

    def device(user, step, split, s, ns, c, counts, nsets, ndim, q, f, stream):
        rows = [ProposalRows(C.cast(s, C.c_void_p).value, ns, ndim, stream)]
        try:
            if split < 0:
                setup(rows[0])
                return
            base = C.cast(c, C.c_void_p).value or 0
            off = 0
            for j in range(nsets):
                n = int(counts[j])
                rows.append(ProposalRows(base + off * ndim * 8, n, ndim, stream))
                off += n
            qo, fo = _proposal_arrays(propose(rows[0], rows[1:], user_random(seed_box[0], step, split)))
            ptrs, streams = [], set()
            for a, want, what in ((qo, (ns, ndim), "q"), (fo, (ns,), "factors")):
                cai = getattr(a, "__cuda_array_interface__", None)
                if cai is None:
                    a = np.ascontiguousarray(a)
                    _check_proposal(a.shape, a.dtype, want, what)
                    ptrs.append((a, a.ctypes.data, a.strides[0] if a.ndim else 8))
                    continue
                _check_proposal(cai["shape"], cai["typestr"], want, what)
                if cai.get("mask") is not None:
                    raise ValueError("masked CUDA arrays are not supported as proposals")
                strides = cai.get("strides")
                if strides is not None and len(want) == 2 and ndim > 1 and strides[1] != 8:
                    raise ValueError("the rows of q must be contiguous; only the first axis may be strided")
                stride = (8 * want[-1] if len(want) == 2 else 8) if strides is None else int(strides[0])
                streams.add((cai["stream"] or 0) if "stream" in cai else EB_STREAM_UNKNOWN)
                ptrs.append((a, cai["data"][0], stride))
            streams.discard(0)
            stream_id = streams.pop() if len(streams) == 1 else (EB_STREAM_UNKNOWN if streams else 0)
            (_, qp, qs), (_, fp, fs) = ptrs
            rc = lib().eb_proposal_result(h, C.c_void_p(qp), int(qs) if ns > 1 else ndim * 8, C.c_void_p(fp),
                                          int(fs) if ns > 1 else 8, int(ns), int(stream_id))
            if rc != EB_OK:
                _raise(rc, lib().eb_last_error(h).decode())
        finally:
            for r in rows:
                r._release()

    def call(*args):
        try:
            if where == EB_CALLBACK_HOST:
                host(*args[:-1])
            else:
                device(*args)
            return 0
        except BaseException as e:  # noqa: B902 -- re-raised unchanged when the ABI call returns
            failure[0] = e
            return 1

    return PROPOSAL_FN(call)


def _host_result(out, m):
    """``out`` as a float64 ``[m]`` array, or the shape / dtype error."""
    a = np.asarray(out)
    if a.shape != (m,):
        raise ValueError("the log-probability function returned shape %s for %d rows; expected (%d,)" % (a.shape, m, m))
    if a.dtype != np.float64:
        raise TypeError("the log-probability function must return float64 values, got %s" % a.dtype)
    return a


def _device_result(h, lp, out, m):
    """Copy a callback's result -- a CUDA-array-interface object or a host array -- into the engine's lp."""
    cai = getattr(out, "__cuda_array_interface__", None)
    if cai is None:
        a = np.ascontiguousarray(_host_result(out, m))
        ptr, stride, stream = a.ctypes.data, 8, 0
    else:
        shape = tuple(cai["shape"])
        if shape != (m,):
            raise ValueError("the log-probability function returned shape %s for %d rows; expected (%d,)" % (shape, m, m))
        if np.dtype(cai["typestr"]) != np.float64:
            raise TypeError("the log-probability function must return float64 values, got %s" % cai["typestr"])
        if cai.get("mask") is not None:
            raise ValueError("masked CUDA arrays are not supported as log-probabilities")
        strides = cai.get("strides")
        # a "stream" entry is the producer's word on ordering (None: none needed); without one (interface v2,
        # which torch exports) the result may still be in flight on any stream, so the engine waits for all
        stream = (cai["stream"] or 0) if "stream" in cai else EB_STREAM_UNKNOWN
        ptr, stride = cai["data"][0], 8 if strides is None else strides[0]
    rc = lib().eb_callback_result(h, lp, C.c_void_p(ptr), int(stride), int(m), int(stream))
    if rc != EB_OK:
        _raise(rc, lib().eb_last_error(h).decode())


def _squeeze(shape):
    """The record shape with its size-1 axes dropped (``ensemble.py:541-545``)."""
    return tuple(int(n) for n in shape if n != 1)


FIXED_WIDTH = (
    "device blobs are fixed-width records: numeric, bool, subarray or structured dtypes; object, string and "
    "ragged blobs are not supported"
)


def _variable_width(dt):
    if dt.hasobject:
        return True
    if dt.subdtype is not None:
        return _variable_width(dt.subdtype[0])
    if dt.fields:
        return any(_variable_width(f[0]) for f in dt.fields.values())
    return dt.kind in "US"  # the reference stores strings as objects (ensemble.py:530-532)


def fixed_width_dtype(dtype, what="blobs_dtype"):
    """``np.dtype(dtype)``, or ``NotImplementedError`` when its records are not plain bytes the engine may copy
    (object pointers, strings)."""
    dt = np.dtype(dtype)
    if _variable_width(dt):
        raise NotImplementedError("%s %s: %s" % (what, dt, FIXED_WIDTH))
    return dt


class BlobSink(object):
    """The blob half of a callback that declares ``blobs_dtype``: checks the records the function returned and
    hands them to the engine (``eb_callback_blobs``).  A layout is ``(dtype, shape)``: one walker's record is an
    array of that dtype and shape, ``record_bytes = dtype.itemsize * prod(shape)``.

    ``expect``: the live layout the records must have (None: any); ``last``: the layout of the records the last
    call delivered, None when it delivered none."""

    def __init__(self, blobs_dtype):
        declared = fixed_width_dtype(blobs_dtype)
        self.dtype = declared.base  # a subarray dtype's shape becomes trailing axes, as np.array(blob, dtype) does
        self.expect = None
        self.last = None

    def layout(self, dtype, shape, m):
        if len(shape) < 1 or shape[0] != m:
            raise ValueError("the function returned blobs of shape %s for %d rows; expected (%d, ...)"
                             % (tuple(shape), m, m))
        if np.dtype(dtype) != self.dtype:
            raise TypeError("the function must return blobs of dtype %s, got %s" % (self.dtype, np.dtype(dtype)))
        lay = (self.dtype, _squeeze(shape[1:]))
        if self.dtype.itemsize * int(np.prod(lay[1], dtype=np.int64)) == 0:
            raise ValueError("the function returned empty blob records")
        if self.expect is not None and lay != self.expect:
            raise ValueError("the function returned blobs of dtype %s and shape %s; the state's blobs have dtype %s "
                             "and shape %s" % (lay[0], lay[1], self.expect[0], self.expect[1]))
        return lay

    def deliver(self, h, blobs, m, device):
        if blobs is None:
            raise ValueError("the log-probability function was declared with blobs_dtype=%s but returned no blobs"
                             % self.dtype)
        cai = getattr(blobs, "__cuda_array_interface__", None) if device else None
        if cai is None:
            a = np.ascontiguousarray(blobs)
            lay = self.layout(a.dtype, a.shape, m)
            rec = a.itemsize * int(np.prod(lay[1], dtype=np.int64))
            ptr, stride, stream = a.ctypes.data, rec, 0
        else:
            if cai.get("mask") is not None:
                raise ValueError("masked CUDA arrays are not supported as blobs")
            dt = np.dtype(cai["descr"]) if cai["typestr"].startswith("|V") and "descr" in cai else np.dtype(cai["typestr"])
            shape = tuple(cai["shape"])
            lay = self.layout(dt, shape, m)
            rec = dt.itemsize * int(np.prod(lay[1], dtype=np.int64))
            strides = cai.get("strides")
            stride = rec
            if strides is not None:
                # a record must be one packed block: the axes after the first C-contiguous (size-1 axes aside)
                inner = [(int(n), int(s)) for n, s in zip(shape[1:], strides[1:]) if n != 1]
                want = dt.itemsize
                for n, s in reversed(inner):
                    if s != want:
                        raise ValueError("blob records must be contiguous; only the first axis may be strided")
                    want *= n
                if m > 1:
                    stride = int(strides[0])
                    if stride < rec:
                        raise ValueError("the blobs' first-axis stride (%d bytes) is shorter than a record (%d bytes)"
                                         % (stride, rec))
            stream = (cai["stream"] or 0) if "stream" in cai else EB_STREAM_UNKNOWN
            ptr = cai["data"][0]
        rc = lib().eb_callback_blobs(h, C.c_void_p(ptr), int(rec), int(stride), int(m), int(stream))
        if rc != EB_OK:
            _raise(rc, lib().eb_last_error(h).decode())
        self.last = lay


def _split_blobs(out):
    """``(lp, blobs)`` of a blob function's result; a result that is not such a pair carries no blobs."""
    if isinstance(out, tuple) and len(out) == 2:
        return out
    return out, None


def make_trampoline(h, evaluate, where, failure, blobs=None):
    """The C callback of one engine: calls ``evaluate`` (host mode: a fresh ``x[m, ndim]`` ndarray the
    function owns; device mode: :class:`DeviceRows`) and writes its result into the engine's ``lp``.
    With a :class:`BlobSink` ``blobs``, ``evaluate`` returns ``(lp, blobs)`` and the records go to the engine
    too.  Any exception is stored as ``failure[0]`` and the engine is told to stop (``EB_ERR_CALLBACK``)."""

    def host(user, x, m, ndim, lp, stream):
        try:
            rows = np.ctypeslib.as_array(x, shape=(m, ndim)).copy()
            out = evaluate(rows)
            if blobs is not None:
                out, b = _split_blobs(out)
                blobs.deliver(h, b, m, False)
            np.ctypeslib.as_array(lp, shape=(m,))[:] = _host_result(out, m)
            return 0
        except BaseException as e:  # noqa: B902 -- re-raised unchanged when the ABI call returns
            failure[0] = e
            return 1

    def device(user, x, m, ndim, lp, stream):
        rows = DeviceRows(C.cast(x, C.c_void_p).value, m, ndim, stream)
        try:
            out = evaluate(rows)
            if blobs is not None:
                out, b = _split_blobs(out)
                blobs.deliver(h, b, m, True)
            _device_result(h, lp, out, m)
            return 0
        except BaseException as e:  # noqa: B902
            failure[0] = e
            return 1
        finally:
            rows._release()

    return LOGPROB_FN(host if where == EB_CALLBACK_HOST else device)


class BatchRows(DeviceRows):
    """The ``[nbatch, m, ndim]`` rows a device-mode batch callback receives (:class:`DeviceRows` otherwise)."""

    __slots__ = ()

    def __init__(self, ptr, nbatch, m, ndim, stream):
        super().__init__(ptr, nbatch * m, ndim, stream)
        self._cai["shape"] = (int(nbatch), int(m), int(ndim))


def _batch_shape_error(shape, K, m, ndim):
    return NotImplementedError(
        "a batched log-probability function receives x[nbatch, m, ndim] = [%d, %d, %d] and must return lp[nbatch, m] "
        "= (%d, %d) float64 values; it returned shape %s" % (K, m, ndim, K, m, tuple(shape)))


def _batch_host_values(out, K, m, ndim):
    """A batched function's host result ``lp[K, m]`` as a float64 ``[K m]`` array, or the shape / dtype error."""
    a = np.asarray(out)
    if a.shape != (K, m):
        raise _batch_shape_error(a.shape, K, m, ndim)
    if a.dtype != np.float64:
        raise TypeError("the log-probability function must return float64 values, got %s" % a.dtype)
    return np.ascontiguousarray(a).reshape(K * m)


def _batch_result(h, lp, out, K, m, ndim):
    """Flatten a device-mode batched function's ``lp[K, m]`` -- a numpy array or a CUDA-array-interface object whose
    rows follow each other at one stride -- into the engine's ``lp[K m]`` (``eb_callback_result``)."""
    cai = getattr(out, "__cuda_array_interface__", None)
    if cai is None:
        a = _batch_host_values(out, K, m, ndim)
        ptr, stride, stream = a.ctypes.data, 8, 0
    else:
        shape = tuple(cai["shape"])
        if shape != (K, m):
            raise _batch_shape_error(shape, K, m, ndim)
        if np.dtype(cai["typestr"]) != np.float64:
            raise TypeError("the log-probability function must return float64 values, got %s" % cai["typestr"])
        if cai.get("mask") is not None:
            raise ValueError("masked CUDA arrays are not supported as log-probabilities")
        strides = cai.get("strides")
        stride = 8
        if strides is not None:
            s0, s1 = int(strides[0]), int(strides[1])
            stride = s1 if m > 1 else s0
            if K > 1 and m > 1 and s0 != m * s1:
                raise ValueError("the log-probabilities lp[nbatch, m] must be one strided run of nbatch * m values "
                                 "(strides %s)" % (tuple(strides),))
        stream = (cai["stream"] or 0) if "stream" in cai else EB_STREAM_UNKNOWN
        ptr = cai["data"][0]
    rc = lib().eb_callback_result(h, lp, C.c_void_p(ptr), int(stride), int(K * m), int(stream))
    if rc != EB_OK:
        _raise(rc, lib().eb_last_error(h).decode())


def make_batch_trampoline(h, fn, where, failure, nbatch):
    """The C callback of a batch engine: the engine's ``[nbatch m, ndim]`` rows go to ``fn`` as ``x[nbatch, m,
    ndim]`` (host mode: a fresh ndarray; device mode: :class:`BatchRows`), and its ``lp[nbatch, m]`` comes back
    flattened.  Exceptions as :func:`make_trampoline`."""

    def host(user, x, rows, ndim, lp, stream):
        try:
            m = rows // nbatch
            out = fn(np.ctypeslib.as_array(x, shape=(rows, ndim)).copy().reshape(nbatch, m, ndim))
            np.ctypeslib.as_array(lp, shape=(rows,))[:] = _batch_host_values(out, nbatch, m, ndim)
            return 0
        except BaseException as e:  # noqa: B902
            failure[0] = e
            return 1

    def device(user, x, rows, ndim, lp, stream):
        m = rows // nbatch
        block = BatchRows(C.cast(x, C.c_void_p).value, nbatch, m, ndim, stream)
        try:
            _batch_result(h, lp, fn(block), nbatch, m, ndim)
            return 0
        except BaseException as e:  # noqa: B902
            failure[0] = e
            return 1
        finally:
            block._release()

    return LOGPROB_FN(host if where == EB_CALLBACK_HOST else device)


class Chain(object):
    """Thin owner of one ``eb_chain``: a stored chain ``[slots, nwalkers, ndim]`` in device memory
    (``emcee_b200.DeviceBackend`` builds on it).  Errors map as in :class:`Engine`, and a device
    allocation that fails or cannot fit raises ``MemoryError``."""

    def __init__(self, nwalkers, ndim, device=0):
        self._h = C.c_void_p()
        self.nwalkers, self.ndim, self.device = int(nwalkers), int(ndim), int(device)
        rc = lib().eb_chain_create(self.device, self.nwalkers, self.ndim, C.byref(self._h))
        if rc != EB_OK:
            msg = lib().eb_chain_last_error(None).decode()
            self._h = C.c_void_p()
            raise (ValueError if rc == EB_ERR_INVALID else EngineError)(msg)

    def _check(self, rc):
        if rc != EB_OK:
            _raise(rc, lib().eb_chain_last_error(self._h).decode())

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().eb_chain_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def grow(self, nslots):
        """Capacity of at least ``nslots`` stored steps (one new segment for the missing ones)."""
        self._check(lib().eb_chain_grow(self._h, int(nslots)))

    def capacity(self):
        """``(slots, device bytes)``."""
        n, b = C.c_uint64(), C.c_uint64()
        self._check(lib().eb_chain_capacity(self._h, C.byref(n), C.byref(b)))
        return int(n.value), int(b.value)

    def write(self, slot, coords, log_prob, accepted=None):
        coords = _f64(coords, (self.nwalkers, self.ndim))
        log_prob = _f64(log_prob, (self.nwalkers,))
        acc = None
        if accepted is not None:
            acc = np.ascontiguousarray(accepted, dtype=np.uint8)
            assert acc.shape == (self.nwalkers,)
        self._check(
            lib().eb_chain_write(
                self._h, int(slot), _as_dp(coords), _as_dp(log_prob),
                None if acc is None else acc.ctypes.data_as(C.POINTER(C.c_uint8)),
            )
        )

    def read(self, first, stride, count, coords=True, log_prob=True):
        """``(coords[count, nwalkers, ndim] or None, log_prob[count, nwalkers] or None)`` of the slots
        ``first + k * stride``."""
        x = np.empty((count, self.nwalkers, self.ndim)) if coords else None
        lp = np.empty((count, self.nwalkers)) if log_prob else None
        self._check(
            lib().eb_chain_read(
                self._h, int(first), int(stride), int(count),
                None if x is None else _as_dp(x), None if lp is None else _as_dp(lp),
            )
        )
        return x, lp

    def read_to(self, first, stride, count, coords_shape=None, log_prob_shape=None):
        """:meth:`read` into new :class:`DeviceArray` s of the given shapes (None: not read), device to device
        (``eb_chain_read_to``); a shape holds ``count * nwalkers * ndim`` or ``count * nwalkers`` values."""
        x = None if coords_shape is None else DeviceArray(coords_shape, self.device)
        lp = None if log_prob_shape is None else DeviceArray(log_prob_shape, self.device)
        self._check(lib().eb_chain_read_to(
            self._h, int(first), int(stride), int(count),
            None if x is None else C.c_void_p(x._ptr), None if lp is None else C.c_void_p(lp._ptr)))
        return x, lp

    def read_segments_to(self, nseg, first, stride, count, coords=True, log_prob=True):
        """:meth:`read_to` in the per-segment layout (``eb_chain_read_segments_to``): the walkers are ``nseg``
        segments of ``nw = nwalkers / nseg``, and the result is ``(coords[nseg, count * nw, ndim] or None,
        log_prob[nseg, count * nw] or None)`` as :class:`DeviceArray` s."""
        nseg = int(nseg)
        nw = self.nwalkers // nseg
        x = DeviceArray((nseg, count * nw, self.ndim), self.device) if coords else None
        lp = DeviceArray((nseg, count * nw), self.device) if log_prob else None
        self._check(lib().eb_chain_read_segments_to(
            self._h, nseg, int(first), int(stride), int(count),
            None if x is None else C.c_void_p(x._ptr), None if lp is None else C.c_void_p(lp._ptr)))
        return x, lp

    def accepted(self):
        out = np.empty(self.nwalkers)
        self._check(lib().eb_chain_accepted(self._h, _as_dp(out)))
        return out

    def autocorr_function(self, first, stride, count, nseg=1):
        """Walker-averaged normalised autocorrelation function ``[count, ndim]`` of the stored slice
        (``eb_chain_autocorr``; the same numbers as :meth:`Engine.autocorr_function` of its host copy).  With
        ``nseg > 1``, one per segment of ``nwalkers / nseg`` walkers: ``[nseg, count, ndim]``, row ``k`` equal to
        the function of segment ``k`` stored alone (``eb_chain_autocorr_segments``)."""
        nseg = int(nseg)
        out = np.empty((nseg, self.ndim, int(count)), dtype=np.float64)
        self._check(lib().eb_chain_autocorr_segments(self._h, nseg, int(first), int(stride), int(count),
                                                     _as_dp(out)))
        out = np.ascontiguousarray(np.swapaxes(out, 1, 2))
        return out[0] if nseg == 1 else out

    def select(self, what, first, stride, count, ranks, nseg=1):
        """``(values[len(ranks), D], has_nan[D], passes)``: the exact order statistics at 0-based ``ranks`` of
        each parameter's ``count * nwalkers`` values in the stored slice (``eb_chain_select``); ``what`` is
        ``"chain"`` (D = ndim) or ``"log_prob"`` (D = 1).  With ``nseg > 1``, those of each segment of
        ``nw = nwalkers / nseg`` walkers (``count * nw`` values): ``(values[nseg, len(ranks), D],
        has_nan[nseg, D], passes)`` (``eb_chain_select_segments``)."""
        nseg = int(nseg)
        ranks = np.ascontiguousarray(ranks, dtype=np.uint64)
        D = self.ndim if what == "chain" else 1
        out = np.empty((nseg, ranks.size, D))
        has_nan = np.zeros((nseg, D), dtype=np.uint8)
        passes = C.c_uint32()
        self._check(lib().eb_chain_select_segments(
            self._h, nseg, EB_CHAIN_COORDS if what == "chain" else EB_CHAIN_LOG_PROB, int(first), int(stride),
            int(count), ranks.ctypes.data_as(C.POINTER(C.c_uint64)), ranks.size, _as_dp(out),
            has_nan.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(passes)))
        if nseg == 1:
            return out[0], has_nan[0].astype(bool), int(passes.value)
        return out, has_nan.astype(bool), int(passes.value)

    def moments(self, first, stride, count, nseg=1):
        """``(mean[ndim], cov[ndim, ndim], n)`` of the stored slice (``eb_chain_moments``).  With ``nseg > 1``,
        those of each segment of ``nwalkers / nseg`` walkers: ``(mean[nseg, ndim], cov[nseg, ndim, ndim], n)``
        with ``n`` the samples of one segment (``eb_chain_moments_segments``)."""
        nseg = int(nseg)
        shape = () if nseg == 1 else (nseg,)
        mean = np.empty(shape + (self.ndim,))
        cov = np.empty(shape + (self.ndim, self.ndim))
        n = C.c_uint64()
        fn = lib().eb_chain_moments if nseg == 1 else lib().eb_chain_moments_segments
        args = () if nseg == 1 else (nseg,)
        self._check(fn(self._h, *args, int(first), int(stride), int(count), _as_dp(mean), _as_dp(cov), C.byref(n)))
        return mean, cov, int(n.value)

    def histogram(self, what, first, stride, count, bins, outer, edges, nseg=1):
        """``hist[D, bins]`` (int64) of the stored slice with numpy's uniform-bin rule (``eb_chain_histogram``):
        ``outer[D, 3]`` holds each column's ``(first_edge, last_edge, norm_denom)``, ``edges[D, bins + 1]`` its
        edges; ``what`` is ``"chain"`` (D = ndim) or ``"log_prob"`` (D = 1).  With ``nseg > 1``, those of each
        segment of ``nwalkers / nseg`` walkers: ``outer[nseg * D, 3]`` and ``edges[nseg * D, bins + 1]`` in column
        order ``k * D + d``, ``hist[nseg * D, bins]`` (``eb_chain_histogram_segments``)."""
        nseg = int(nseg)
        D = nseg * (self.ndim if what == "chain" else 1)
        bins = int(bins)
        outer = _f64(outer, (D, 3))
        edges = _f64(edges, (D, bins + 1))
        hist = np.empty((D, bins), dtype=np.uint64)
        self._check(lib().eb_chain_histogram_segments(
            self._h, nseg, EB_CHAIN_COORDS if what == "chain" else EB_CHAIN_LOG_PROB, int(first), int(stride),
            int(count), bins, _as_dp(outer), _as_dp(edges), hist.ctypes.data_as(C.POINTER(C.c_uint64))))
        return hist.astype(np.int64)

    def histogram2d(self, first, stride, count, params, bins, edges, nseg=1):
        """``hist[npairs, bins, bins]`` (uint64) of every pair of ``itertools.combinations(params, 2)`` with
        ``np.histogramdd``'s rule against ``edges[len(params), bins + 1]`` (``eb_chain_histogram2d``).  With
        ``nseg > 1``, those of each segment of ``nwalkers / nseg`` walkers: ``edges[nseg * len(params), bins + 1]``
        (segment-major), ``hist[nseg, npairs, bins, bins]`` (``eb_chain_histogram2d_segments``)."""
        nseg = int(nseg)
        params = np.ascontiguousarray(params, dtype=np.uint32)
        m, bins = params.size, int(bins)
        edges = _f64(edges, (nseg * m, bins + 1))
        hist = np.empty(((nseg,) if nseg > 1 else ()) + (m * (m - 1) // 2, bins, bins), dtype=np.uint64)
        self._check(lib().eb_chain_histogram2d_segments(
            self._h, nseg, int(first), int(stride), int(count), params.ctypes.data_as(C.POINTER(C.c_uint32)), m,
            bins, _as_dp(edges), hist.ctypes.data_as(C.POINTER(C.c_uint64))))
        return hist


class RingChain(Chain):
    """A :class:`Chain` reader over an engine's running window (``eb_window_chain``): the ring belongs to the engine,
    which this object keeps alive; :meth:`close` releases nothing."""

    def __init__(self, engine, handle):
        self._engine = engine
        self._h = handle
        self.nwalkers, self.ndim, self.device = engine.nwalkers, engine.ndim, engine.device

    def close(self):
        pass


class Engine(object):
    """Thin owner of one ``eb_ctx``.  Maps error codes onto the exception types
    the reference raises for the same conditions (``ensemble.py:314-323,
    357-358,476-479,550-551``; ``moves/red_blue.py:64-70``)."""

    def __init__(self, nwalkers, ndim, seed, device=0):
        self._h = C.c_void_p()
        self._cb = None  # the registered C callback (kept alive while the engine may call it)
        self._cb_failure = [None]
        self._blob_sink = None  # BlobSink of a callback that declares blobs_dtype
        self._blob_layout = None  # (dtype, shape) of the state's blob records, or None
        self._props = {}  # slot -> the registered C proposal function (kept alive while the engine may call it)
        self._seed_box = [int(seed) & (2**64 - 1)]  # the Philox key, read by the proposal trampolines
        self.nwalkers, self.ndim, self.device = int(nwalkers), int(ndim), int(device)
        rc = lib().eb_create(self.device, self.nwalkers, self.ndim, int(seed) & (2**64 - 1), C.byref(self._h))
        if rc != EB_OK:
            msg = lib().eb_last_error(None).decode()
            self._h = C.c_void_p()
            raise (ValueError if rc == EB_ERR_INVALID else EngineError)(msg)

    # -- plumbing -------------------------------------------------------------
    def _check(self, rc):
        if rc == EB_ERR_CALLBACK:
            exc, self._cb_failure[0] = self._cb_failure[0], None
            if exc is not None:
                raise exc  # the caller's own exception, with its traceback
        if rc != EB_OK:
            _raise(rc, lib().eb_last_error(self._h).decode())

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().eb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- model / state ----------------------------------------------------------
    def set_model(self, kind, params):
        params = _f64(np.asarray(params, dtype=np.float64).ravel())
        self._check(lib().eb_model_set(self._h, MODEL_KINDS[kind], _as_dp(params), params.size))

    def set_bounds(self, lower=None, upper=None):
        """The prior's support ``lower <= x <= upper`` (``eb_model_set_bounds``): outside it the
        log-probability is ``-inf``.  ``None, None`` clears it; ``set_model`` clears it too."""
        if lower is None and upper is None:
            self._check(lib().eb_model_set_bounds(self._h, None, None))
            return
        lo = _f64(np.asarray(lower, dtype=np.float64).ravel(), (self.ndim,))
        hi = _f64(np.asarray(upper, dtype=np.float64).ravel(), (self.ndim,))
        self._check(lib().eb_model_set_bounds(self._h, _as_dp(lo), _as_dp(hi)))

    def set_callback(self, evaluate, where, blobs_dtype=None):
        """Make ``evaluate`` the model (``eb_model_set_callback``): called once per half-step with the
        split's proposals, ``where`` = ``"host"`` (a fresh ``[m, ndim]`` ndarray) or ``"device"``
        (:class:`DeviceRows`).  Its exceptions propagate unchanged from the call that ran it.  With
        ``blobs_dtype``, ``evaluate`` returns ``(lp, blobs)`` and the engine carries the blobs."""
        mode = {"host": EB_CALLBACK_HOST, "device": EB_CALLBACK_DEVICE}[where]
        sink = None if blobs_dtype is None else BlobSink(blobs_dtype)
        cb = make_trampoline(self._h, evaluate, mode, self._cb_failure, sink)
        self._check(lib().eb_model_set_callback(self._h, cb, None, mode))
        self._cb = cb
        self._blob_sink = sink
        self._blob_layout = None

    def set_graphs(self, specs, keep):
        """Make captured graphs the model (``eb_model_set_graphs``): ``specs`` holds one
        ``(m, exec, x_ptr, x_row_stride, lp_ptr, lp_stride)`` per row count; ``keep`` (the graphs' owners) stays
        referenced while they are the model."""
        arr = (EbGraph * len(specs))()
        for k, (m, ex, xp, xs, lpp, lps) in enumerate(specs):
            arr[k].m, arr[k].exec = int(m), int(ex)
            arr[k].x, arr[k].x_row_stride_bytes = int(xp), int(xs)
            arr[k].lp, arr[k].lp_stride_bytes = int(lpp), int(lps)
        self._check(lib().eb_model_set_graphs(self._h, arr, len(specs)))
        self._cb = list(keep)
        self._blob_sink = None
        self._blob_layout = None

    def _expect_blobs(self):
        if self._blob_sink is not None:
            self._blob_sink.expect = self._blob_layout
            self._blob_sink.last = None

    def set_state(self, coords, log_prob=None, blobs=None):
        """Upload the state.  ``log_prob=None``: evaluated by the model, and a blob function's records become
        the state's blobs.  Otherwise ``blobs`` (``[nwalkers, ...]``, or None) are the state's blobs: they must
        have the dtype the function declared, and are checked before anything is uploaded -- the engine copies
        them as raw bytes."""
        coords = _f64(coords, (self.nwalkers, self.ndim))
        lp = None if log_prob is None else _f64(log_prob, (self.nwalkers,))
        if blobs is not None:
            if self._blob_sink is None:
                raise NotImplementedError("the state carries blobs, but the log-probability function declares none")
            blobs = np.asarray(blobs)
            fixed_width_dtype(blobs.dtype, "the state's blobs have dtype")
            if blobs.dtype != self._blob_sink.dtype:
                raise ValueError("the state's blobs have dtype %s; the function declares %s"
                                 % (blobs.dtype, self._blob_sink.dtype))
            blobs = np.ascontiguousarray(blobs)
            if blobs.ndim < 1 or blobs.shape[0] != self.nwalkers:
                raise ValueError("invalid blobs size; expected {0}".format(self.nwalkers))
            if blobs.nbytes == 0:
                raise ValueError("the state's blob records are empty")
        self._blob_layout = None
        self._expect_blobs()
        self._check(lib().eb_set_state(self._h, _as_dp(coords), None if lp is None else _as_dp(lp)))
        if lp is None:
            self._blob_layout = None if self._blob_sink is None else self._blob_sink.last
        elif blobs is not None:
            self._check(lib().eb_set_state_blobs(self._h, C.c_void_p(blobs.ctypes.data), blobs.nbytes // self.nwalkers))
            self._blob_layout = (blobs.dtype, _squeeze(blobs.shape[1:]))

    def set_state_from(self, coords, log_prob=None):
        """:meth:`set_state` from device memory (``eb_set_state_from``): ``coords`` and ``log_prob`` (or None) are
        :class:`CudaRows`; the copy waits for the producers' stream.  ``log_prob=None``: evaluated by the model,
        and a blob function's records become the state's blobs."""
        stream = _one_stream(coords.stream, 0 if log_prob is None else log_prob.stream)
        self._blob_layout = None
        self._expect_blobs()
        self._check(lib().eb_set_state_from(
            self._h, C.c_void_p(coords.ptr), coords.stride, None if log_prob is None else C.c_void_p(log_prob.ptr),
            8 if log_prob is None else log_prob.stride, stream))
        if log_prob is None:
            self._blob_layout = None if self._blob_sink is None else self._blob_sink.last

    def get_state_to(self):
        """``(coords, log_prob)`` of the live state as new :class:`DeviceArray` s (``eb_get_state_to``)."""
        x = DeviceArray((self.nwalkers, self.ndim), self.device)
        lp = DeviceArray((self.nwalkers,), self.device)
        self._check(lib().eb_get_state_to(self._h, C.c_void_p(x._ptr), C.c_void_p(lp._ptr)))
        return x, lp

    def get_blobs(self):
        """The state's blobs ``[nwalkers, *shape]`` (a fresh array), or None when it has none."""
        if self._blob_layout is None:
            return None
        dt, shape = self._blob_layout
        out = np.empty((self.nwalkers,) + shape, dtype=dt)
        self._check(lib().eb_get_blobs(self._h, C.c_void_p(out.ctypes.data)))
        return out

    def get_state(self, coords=None, log_prob=None):
        """Device -> host copy of the live state, into fresh arrays or into the
        given (C-contiguous float64, e.g. pinned) buffers."""
        coords = np.empty((self.nwalkers, self.ndim), dtype=np.float64) if coords is None else coords
        lp = np.empty(self.nwalkers, dtype=np.float64) if log_prob is None else log_prob
        assert coords.flags.c_contiguous and coords.dtype == np.float64 and coords.shape == (self.nwalkers, self.ndim)
        assert lp.flags.c_contiguous and lp.dtype == np.float64 and lp.shape == (self.nwalkers,)
        self._check(lib().eb_get_state(self._h, _as_dp(coords), _as_dp(lp)))
        return coords, lp

    def owned_rows(self):
        """``(row0, nrows)`` of the walkers this engine updates (all of them on one GPU)."""
        r0, n = C.c_int64(), C.c_int64()
        self._check(lib().eb_owned_rows(self._h, C.byref(r0), C.byref(n)))
        return int(r0.value), int(n.value)

    def get_state_rows(self, row0, nrows, coords, log_prob):
        """Device -> host copy of rows ``[row0, row0 + nrows)`` into the matching
        row slices of the full-size host arrays ``coords`` / ``log_prob`` (not collective)."""
        assert coords.flags.c_contiguous and coords.dtype == np.float64 and coords.shape == (self.nwalkers, self.ndim)
        assert log_prob.flags.c_contiguous and log_prob.dtype == np.float64 and log_prob.shape == (self.nwalkers,)
        c, lp = coords[row0 : row0 + nrows], log_prob[row0 : row0 + nrows]
        self._check(lib().eb_get_state_rows(self._h, int(row0), int(nrows), _as_dp(c), _as_dp(lp)))
        return coords, log_prob

    def moments(self):
        """``(mean[D], cov[D, D], count, naccepted_total)`` of the samples folded in so far
        (option ``moments_every``); per rank on a sharded ensemble."""
        mean = np.empty(self.ndim)
        cov = np.empty((self.ndim, self.ndim))
        n, na = C.c_uint64(), C.c_uint64()
        self._check(lib().eb_moments(self._h, _as_dp(mean), _as_dp(cov), C.byref(n), C.byref(na)))
        return mean, cov, int(n.value), int(na.value)

    def histograms_config(self, every, bins, outer, edges, log_prob=False, params2d=None, bins2d=0, edges2d=None):
        """Count every ``every``-th step into running histograms (``eb_histograms_config``; zeroes the counts):
        ``outer[ndim + log_prob, 3]`` / ``edges[ndim + log_prob, bins + 1]`` as :meth:`Chain.histogram` takes them,
        the log-probabilities in the last row; ``params2d`` (or None) with ``edges2d[len(params2d), bins2d + 1]``."""
        rows, bins = self.ndim + (1 if log_prob else 0), int(bins)
        outer = _f64(outer, (rows, 3))
        edges = _f64(edges, (rows, bins + 1))
        p, m, e2 = None, 0, None
        if params2d is not None:
            params2d = np.ascontiguousarray(params2d, dtype=np.uint32)
            m, bins2d = params2d.size, int(bins2d)
            e2 = _f64(edges2d, (m, bins2d + 1))
            p = params2d.ctypes.data_as(C.POINTER(C.c_uint32))
        self._check(lib().eb_histograms_config(
            self._h, int(every), bins, _as_dp(outer), _as_dp(edges), int(bool(log_prob)), p, m, int(bins2d),
            None if e2 is None else _as_dp(e2)))
        self._hist_shape = (rows, bins, m, int(bins2d))

    def histograms(self, counts=True):
        """``(hist[ndim + log_prob, bins] uint64, hist2d[npairs, bins2d, bins2d] uint64 or None, count)`` of the
        running histograms (``eb_histograms``); ``counts=False`` reads only ``count``."""
        rows, bins, m, bins2d = getattr(self, "_hist_shape", (self.ndim, 1, 0, 0))
        hist = np.zeros((rows, bins), dtype=np.uint64) if counts else None
        hist2 = np.zeros((m * (m - 1) // 2, bins2d, bins2d), dtype=np.uint64) if m and counts else None
        n = C.c_uint64()
        self._check(lib().eb_histograms(
            self._h, None if hist is None else hist.ctypes.data_as(C.POINTER(C.c_uint64)),
            None if hist2 is None else hist2.ctypes.data_as(C.POINTER(C.c_uint64)), C.byref(n)))
        return hist, hist2, int(n.value)

    def trace_config(self, every):
        """Record one row of ensemble statistics after every ``every``-th step (``eb_trace_config``)."""
        self._check(lib().eb_trace_config(self._h, int(every)))

    def trace_count(self):
        n = C.c_uint64()
        self._check(lib().eb_trace_count(self._h, C.byref(n)))
        return int(n.value)

    def trace_read(self, first=0):
        """``(step[n] uint64, rows[n, 2 ndim + 4])`` of the recorded rows from ``first`` on (``eb_trace_read``)."""
        n = max(self.trace_count() - int(first), 0)
        step = np.zeros(n, dtype=np.uint64)
        rows = np.zeros((n, 2 * self.ndim + 4), dtype=np.float64)
        if n:
            self._check(lib().eb_trace_read(self._h, int(first), n, step.ctypes.data_as(C.POINTER(C.c_uint64)),
                                            _as_dp(rows)))
        return step, rows

    def trace_best(self):
        """``(coords[ndim], log_prob, step, walker)`` of ``eb_trace_best``."""
        coords = np.zeros(self.ndim, dtype=np.float64)
        lp, step, walker = C.c_double(), C.c_uint64(), C.c_uint64()
        self._check(lib().eb_trace_best(self._h, _as_dp(coords), C.byref(lp), C.byref(step), C.byref(walker)))
        return coords, float(lp.value), int(step.value), int(walker.value)

    def reservoir_config(self, size, every):
        """Keep ``size`` of the rows of every ``every``-th step (``eb_reservoir_config``).  Values past uint64 reach the
        library as its largest value instead of wrapping: a size it refuses, a cadence no run reaches."""
        top = 2**64 - 1
        self._check(lib().eb_reservoir_config(self._h, min(int(size), top), min(int(every), top)))

    def reservoir_count(self):
        """``(offered, kept)`` rows of the reservoir (``eb_reservoir_count``)."""
        offered, kept = C.c_uint64(), C.c_uint64()
        self._check(lib().eb_reservoir_count(self._h, C.byref(offered), C.byref(kept)))
        return int(offered.value), int(kept.value)

    def reservoir_read(self, cuda=False):
        """``(coords[k, ndim], log_prob[k], step[k] uint64, walker[k] int64)`` of the kept rows in the reservoir's
        order (``eb_reservoir_read``); ``cuda=True``: coords and log_prob as :class:`DeviceArray` s
        (``eb_reservoir_read_to``)."""
        k = self.reservoir_count()[1]
        step = np.zeros(k, dtype=np.uint64)
        walker = np.zeros(k, dtype=np.int64)
        sp, wp = step.ctypes.data_as(C.POINTER(C.c_uint64)), walker.ctypes.data_as(C.POINTER(C.c_int64))
        if cuda:
            coords, lp = DeviceArray((k, self.ndim), self.device), DeviceArray((k,), self.device)
            self._check(lib().eb_reservoir_read_to(self._h, C.c_void_p(coords._ptr), C.c_void_p(lp._ptr), sp, wp))
        else:
            coords, lp = np.zeros((k, self.ndim), dtype=np.float64), np.zeros(k, dtype=np.float64)
            self._check(lib().eb_reservoir_read(self._h, _as_dp(coords), _as_dp(lp), sp, wp))
        return coords, lp, step, walker

    def running_acf_config(self, max_lag, every):
        """Lag sums up to ``max_lag`` of every ``every``-th step (``eb_running_acf_config``).  Values past uint64
        reach the library as its largest value instead of wrapping: lags it cannot hold, a cadence no run reaches."""
        top = 2**64 - 1
        self._check(lib().eb_running_acf_config(self._h, min(int(max_lag), top), min(int(every), top)))

    def running_acf_count(self):
        """Steps recorded into the running autocorrelation (``eb_running_acf_count``)."""
        n = C.c_uint64()
        self._check(lib().eb_running_acf_count(self._h, C.byref(n)))
        return int(n.value)

    def running_acf_read(self, max_lag):
        """``rho[min(n, max_lag + 1), ndim]`` of the recorded steps (``eb_running_acf_read``)."""
        rho = np.zeros((min(self.running_acf_count(), int(max_lag) + 1), self.ndim), dtype=np.float64)
        self._check(lib().eb_running_acf_read(self._h, _as_dp(rho)))
        return rho

    def window_config(self, size, every):
        """Keep the last ``size`` states of every ``every``-th step (``eb_window_config``).  Values past uint64 reach
        the library as its largest value instead of wrapping: a size it cannot allocate, a cadence no run reaches."""
        top = 2**64 - 1
        self._check(lib().eb_window_config(self._h, min(int(size), top), min(int(every), top)))

    def window_count(self):
        """``(recorded, filled)`` of the running window (``eb_window_count``)."""
        recorded, filled = C.c_uint64(), C.c_uint64()
        self._check(lib().eb_window_count(self._h, C.byref(recorded), C.byref(filled)))
        return int(recorded.value), int(filled.value)

    def window_steps(self):
        """``(steps[filled], seeds[filled])`` (uint64) of the window's slots, oldest first (``eb_window_steps``)."""
        n = self.window_count()[1]
        steps, seeds = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64)
        self._check(lib().eb_window_steps(self._h, steps.ctypes.data_as(C.POINTER(C.c_uint64)),
                                          seeds.ctypes.data_as(C.POINTER(C.c_uint64))))
        return steps, seeds

    def window_chain(self):
        """A :class:`RingChain` over the window's ring (``eb_window_chain``), current as of this call."""
        h = C.c_void_p()
        self._check(lib().eb_window_chain(self._h, C.byref(h)))
        return RingChain(self, h)

    def walkers_gram(self, coords):
        """``(gram[D, D], flags)`` of ``eb_walkers_gram`` for ``coords[rows, D]``."""
        coords = _f64(coords)
        if coords.ndim != 2 or coords.shape[1] != self.ndim:
            raise ValueError("incompatible input dimensions {0}".format(coords.shape))
        gram = np.empty((self.ndim, self.ndim))
        flags = C.c_int()
        self._check(lib().eb_walkers_gram(self._h, _as_dp(coords), coords.shape[0], _as_dp(gram), C.byref(flags)))
        return gram, int(flags.value)

    def autocorr_function(self, chain):
        """Walker-averaged normalised autocorrelation function ``[n_step, n_param]`` of
        ``chain[n_step, n_walker, n_param]`` (``eb_autocorr``)."""
        chain = _f64(chain)
        if chain.ndim != 3:
            raise ValueError("invalid dimensions")
        n_t, n_w, n_d = chain.shape
        out = np.empty((n_d, n_t), dtype=np.float64)
        self._check(lib().eb_autocorr(self._h, _as_dp(chain), n_t, n_w, n_d, _as_dp(out)))
        return np.ascontiguousarray(out.T)

    def compute_log_prob(self, coords):
        coords = _f64(coords)
        if coords.shape[-1] != self.ndim:
            raise ValueError("incompatible input dimensions {0}".format(coords.shape))
        flat = coords.reshape(-1, self.ndim)
        out = np.empty(flat.shape[0], dtype=np.float64)
        self._check(lib().eb_compute_log_prob(self._h, _as_dp(flat), flat.shape[0], _as_dp(out)))
        return out.reshape(coords.shape[:-1])

    def compute_log_prob_from(self, coords):
        """:meth:`compute_log_prob` of a CUDA array ``coords[m, ndim]`` into a new :class:`DeviceArray` ``[m]``
        (``eb_compute_log_prob_from``)."""
        shape = tuple(int(n) for n in coords.__cuda_array_interface__["shape"])
        if len(shape) != 2 or shape[1] != self.ndim:
            raise ValueError("incompatible input dimensions {0}".format(shape))
        rows = CudaRows(coords, shape, self.device, "coords")
        out = DeviceArray((shape[0],), self.device)
        self._check(lib().eb_compute_log_prob_from(self._h, C.c_void_p(rows.ptr), rows.stride, shape[0],
                                                   C.c_void_p(out._ptr), rows.stream))
        return out

    def compute_log_prob_blobs(self, coords):
        """``(log_prob[...], blobs[..., *shape] or None)`` of a blob function for ``coords[..., ndim]``."""
        coords = _f64(coords)
        if coords.shape[-1] != self.ndim:
            raise ValueError("incompatible input dimensions {0}".format(coords.shape))
        flat = coords.reshape(-1, self.ndim)
        m = flat.shape[0]
        out = np.empty(m, dtype=np.float64)
        ptr, nbytes = C.c_void_p(), C.c_size_t()
        self._expect_blobs()
        self._check(lib().eb_compute_log_prob_blobs(self._h, _as_dp(flat), m, _as_dp(out), C.byref(ptr),
                                                    C.byref(nbytes)))
        blobs = None
        if ptr.value:
            try:
                dt, shape = self._blob_sink.last
                raw = (C.c_char * (m * nbytes.value)).from_address(ptr.value)
                blobs = np.frombuffer(raw, dtype=dt).reshape((m,) + shape).copy()
            finally:
                lib().eb_host_free(ptr)
            blobs = blobs.reshape(coords.shape[:-1] + shape)
        return out.reshape(coords.shape[:-1]), blobs

    # -- rng -----------------------------------------------------------------
    def set_rng(self, seed, step):
        self._check(lib().eb_set_rng(self._h, int(seed) & (2**64 - 1), int(step)))
        self._seed_box[0] = int(seed) & (2**64 - 1)

    def set_proposal(self, slot, propose, where, setup=None):
        """Make ``propose(s, c, random) -> (q, factors)`` proposal slot ``slot`` (``eb_move_set_proposal``), called
        once per half-step of a schedule entry of kind ``"user"`` / ``"user_mh"`` whose ``p0`` is ``slot``;
        ``where`` = ``"host"`` (numpy arrays) or ``"device"`` (:class:`ProposalRows`).  ``setup(coords)``, if given,
        is called once per step before the splits of a ``"user"`` entry with ``mode`` 1.  Exceptions propagate
        unchanged from the call that ran the function."""
        mode = {"host": EB_CALLBACK_HOST, "device": EB_CALLBACK_DEVICE}[where]
        fn = make_proposal_trampoline(self._h, propose, setup, mode, self._cb_failure, self._seed_box)
        self._check(lib().eb_move_set_proposal(self._h, int(slot), fn, None, mode))
        self._props[int(slot)] = fn

    def set_proposal_graphs(self, slot, draw, ndraws, specs, keep):
        """Make captured graphs proposal slot ``slot`` (``eb_move_set_proposal_graphs``): ``specs`` holds one
        ``(split, ns, exec, s, s_stride, c, c_stride, draws, draws_stride, q, q_stride, factors, factors_stride)`` per
        split, pointers and byte strides; ``draw`` is ``"uniform"`` or ``"normal"``; ``keep`` (the captures' owners)
        stays referenced while the slot is set."""
        arr = (EbProposalGraph * len(specs))()
        for k, spec in enumerate(specs):
            for name, v in zip([f[0] for f in EbProposalGraph._fields_], spec):
                setattr(arr[k], name, int(v))
        self._check(lib().eb_move_set_proposal_graphs(self._h, int(slot), EB_DRAW_KINDS[draw], int(ndraws), arr,
                                                      len(specs)))
        self._props[int(slot)] = list(keep)

    def get_rng(self):
        seed, step = C.c_uint64(), C.c_uint64()
        self._check(lib().eb_get_rng(self._h, C.byref(seed), C.byref(step)))
        return int(seed.value), int(step.value)

    # -- stepping ----------------------------------------------------------------
    @staticmethod
    def pack_moves(moves):
        """``moves``: list of (descriptor dict, weight)."""
        arr = (EbMove * len(moves))()
        for k, (d, w) in enumerate(moves):
            arr[k].kind = MOVE_KINDS[d["kind"]]
            arr[k].nsplits = int(d["nsplits"])
            arr[k].randomize_split = int(bool(d["randomize_split"]))
            arr[k].live_dangerously = int(bool(d["live_dangerously"]))
            arr[k].weight = float(w)
            arr[k].p0 = float(d["p0"])
            arr[k].p1 = float(d["p1"])
            if d.get("cov") is not None:  # GaussianMove: the array must outlive the call -> kept on `arr`
                cov = np.ascontiguousarray(d["cov"], dtype=np.float64)
                keep = getattr(arr, "_keep", [])
                keep.append(cov)
                arr._keep = keep
                arr[k].cov = cov.ctypes.data_as(_dp)
                arr[k].ncov = cov.size
                arr[k].mode = int(d.get("mode", 0))
                arr[k].seq_index = int(d.get("seq_index", 0))
            elif d["kind"] == "user":
                arr[k].mode = int(d.get("mode", 0))  # EB_USER_SETUP
        return arr

    def move_picks(self, nmoves):
        """How many steps of the last stepping call ran each schedule entry."""
        out = np.zeros(int(nmoves), dtype=np.uint64)
        self._check(lib().eb_move_picks(self._h, out.ctypes.data_as(C.POINTER(C.c_uint64)), int(nmoves)))
        return out

    def step(self, moves, nsteps, want_accepted=True):
        arr = self.pack_moves(moves)
        self._expect_blobs()
        acc = np.zeros(self.nwalkers, dtype=np.uint8) if want_accepted else None
        self._check(
            lib().eb_step(
                self._h, arr, len(arr), int(nsteps),
                None if acc is None else acc.ctypes.data_as(C.POINTER(C.c_uint8)),
            )
        )
        return None if acc is None else acc.astype(bool)

    def step_store(self, moves, nsteps, thin_by, chain, log_prob, accepted, blobs=None):
        """``blobs`` (``[nstore, nwalkers, ...]`` C-contiguous, the state's record layout, or None) gets the
        blobs of the stored steps."""
        arr = self.pack_moves(moves)
        assert chain.flags.c_contiguous and log_prob.flags.c_contiguous and accepted.flags.c_contiguous
        assert chain.dtype == np.float64 and log_prob.dtype == np.float64 and accepted.dtype == np.float64
        self._expect_blobs()
        if blobs is None:
            self._check(
                lib().eb_step_store(
                    self._h, arr, len(arr), int(nsteps), int(thin_by),
                    _as_dp(chain), _as_dp(log_prob), _as_dp(accepted),
                )
            )
            return
        dt, shape = self._blob_layout
        nstore = int(nsteps) // int(thin_by)
        if not blobs.flags.c_contiguous or blobs.nbytes != nstore * self.nwalkers * dt.itemsize * int(np.prod(shape)):
            raise ValueError("the blob store does not match the state's blob records")
        self._check(
            lib().eb_step_store_blobs(
                self._h, arr, len(arr), int(nsteps), int(thin_by),
                _as_dp(chain), _as_dp(log_prob), _as_dp(accepted), C.c_void_p(blobs.ctypes.data),
            )
        )

    def step_store_chain(self, moves, nsteps, thin_by, chain, slot0):
        """Like :meth:`step_store`, into slots ``slot0, slot0 + 1, ...`` of the device
        :class:`Chain` ``chain``."""
        arr = self.pack_moves(moves)
        self._check(lib().eb_step_store_chain(self._h, arr, len(arr), int(nsteps), int(thin_by), chain._h, int(slot0)))

    def naccepted(self):
        out = np.zeros(self.nwalkers, dtype=np.uint64)
        self._check(lib().eb_get_naccepted(self._h, out.ctypes.data_as(C.POINTER(C.c_uint64))))
        return out

    def reset_counters(self):
        self._check(lib().eb_reset_counters(self._h))

    def last_step_timing(self):
        ms, n = C.c_double(), C.c_uint64()
        self._check(lib().eb_last_step_timing(self._h, C.byref(ms), C.byref(n)))
        return float(ms.value), int(n.value)

    def last_kernel_name(self):
        return lib().eb_last_kernel_name(self._h).decode()

    def last_kernel_variant(self):
        """The cell of that kernel the last half-step launch ran (``eb_last_kernel_variant``),
        e.g. ``"tma_rows R=8 epl=8 own_reg=1 warps=16"``."""
        return lib().eb_last_kernel_variant(self._h).decode()

    def set_option(self, name, value):
        self._check(lib().eb_set_option(self._h, name.encode(), int(value)))

    def debug_taps(self):
        n = self.nwalkers
        partners = np.empty((3, n), dtype=np.int64)
        scalar = np.empty(n, dtype=np.float64)
        u = np.empty(n, dtype=np.float64)
        active = np.empty(n, dtype=np.int64)
        cnt = C.c_int64()
        i64 = C.POINTER(C.c_int64)
        self._check(
            lib().eb_debug_taps(
                self._h, partners.ctypes.data_as(i64), _as_dp(scalar), _as_dp(u),
                active.ctypes.data_as(i64), C.byref(cnt),
            )
        )
        k = int(cnt.value)
        return dict(partners=partners[:, :k], scalar=scalar[:k], u_accept=u[:k], active=active[:k])

    def debug_timeline(self):
        """[SM, consumer, tile, event] cycle stamps of the last dense_dmma half-step."""
        buf = np.zeros(1 << 21, dtype=np.int64)
        n = C.c_size_t()
        self._check(lib().eb_debug_timeline(self._h, buf.ctypes.data_as(C.POINTER(C.c_int64)), buf.size, C.byref(n)))
        return buf[: n.value].reshape(-1, 8, 8, 12)  # events 0..5, 9 consumer; 6..8, 10, 11 producer (dense_dmma.cu)

    # -- multi-GPU ---------------------------------------------------------------
    @staticmethod
    def comm_id():
        buf = C.create_string_buffer(EB_COMM_ID_BYTES)
        rc = lib().eb_comm_id(buf)
        if rc != EB_OK:
            raise EngineError("eb_comm_id failed (is libnccl.so.2 loadable?)")
        return buf.raw

    def comm_init(self, comm_id, rank, nranks, mode=EB_COMM_ALLGATHER):
        assert len(comm_id) == EB_COMM_ID_BYTES
        self._check(lib().eb_comm_init(self._h, comm_id, int(rank), int(nranks), int(mode)))

    def comm_export(self):
        buf = C.create_string_buffer(EB_IPC_BLOB_BYTES)
        self._check(lib().eb_comm_export(self._h, buf))
        return buf.raw

    def comm_probe(self, peer, what):
        out = C.c_double()
        self._check(lib().eb_comm_probe(self._h, int(peer), int(what), C.byref(out)))
        return float(out.value)

    def comm_import(self, blobs):
        self._check(lib().eb_comm_import(self._h, blobs))


class BatchEngine(Engine):
    """Thin owner of a batch ``eb_ctx`` (``eb_create_batch``): ``nbatch`` ensembles of ``ens_walkers`` walkers
    stacked as its ``nwalkers = nbatch * ens_walkers`` rows, so every row-wise method of :class:`Engine` takes and
    returns the stacked rows."""

    def __init__(self, nbatch, nwalkers, ndim, seeds, device=0):
        self._h = C.c_void_p()
        self._cb = None
        self._cb_failure = [None]
        self._blob_sink = None
        self._blob_layout = None
        self._props = {}
        self.nbatch, self.ens_walkers = int(nbatch), int(nwalkers)
        self.nwalkers, self.ndim, self.device = self.nbatch * self.ens_walkers, int(ndim), int(device)
        seeds = np.ascontiguousarray(seeds, dtype=np.uint64)
        rc = lib().eb_create_batch(self.device, self.nbatch, self.ens_walkers, self.ndim,
                                   seeds.ctypes.data_as(C.POINTER(C.c_uint64)), C.byref(self._h))
        if rc != EB_OK:
            msg = lib().eb_last_error(None).decode()
            self._h = C.c_void_p()
            _raise(rc, msg)

    def set_callback(self, fn, where):
        """Make ``fn(x[nbatch, m, ndim]) -> lp[nbatch, m]`` the model, called once per half-step for every
        ensemble; ``where`` as :meth:`Engine.set_callback`."""
        mode = {"host": EB_CALLBACK_HOST, "device": EB_CALLBACK_DEVICE}[where]
        cb = make_batch_trampoline(self._h, fn, mode, self._cb_failure, self.nbatch)
        self._check(lib().eb_model_set_callback(self._h, cb, None, mode))
        self._cb = cb

    def get_rng(self):
        """``(seeds[nbatch] uint64, step)``."""
        seeds, step = np.zeros(self.nbatch, dtype=np.uint64), C.c_uint64()
        self._check(lib().eb_batch_rng_get(self._h, seeds.ctypes.data_as(C.POINTER(C.c_uint64)), C.byref(step)))
        return seeds, int(step.value)

    def set_rng(self, seeds, step):
        seeds = np.ascontiguousarray(seeds, dtype=np.uint64)
        if seeds.shape != (self.nbatch,):
            raise ValueError("expected %d seeds, got shape %s" % (self.nbatch, seeds.shape))
        self._check(lib().eb_batch_rng_set(self._h, seeds.ctypes.data_as(C.POINTER(C.c_uint64)), int(step)))
