"""Blobs of user log-probability functions on the GPU: the engine selects each walker's blob record on
the device at accept (``moves/move.py:36-43``) and stores it with the chain (``backends/backend.py:157-231``).

* a blob that is a pure function of the row: every stored and every yielded blob equals f(coords), bit for
  bit, for every move, host mode, device mode with numpy results and with torch tensors (a strided first
  axis), odd nwalkers, several split counts and ndims;
* twin runs with and without blobs: identical coords, log_prob, accept counts and function inputs;
* record sizes that reach every copy width of the select kernel and its byte path;
* the reference's ``test_blob_mismatch`` flow and the other edges: missing blobs, a given log_prob without
  blobs, a State whose blobs are objects or another dtype, ``DeviceBackend``, thinning, ``store=False``, ``iterations=0``, resuming after an exception,
  pickling, ``compute_log_prob``;
* torch CUDA-array blobs written late on a side stream (v3 and v2) and with a strided first axis;
* 65 536 x 128 at scale.
"""
import pickle

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import models, moves

pytestmark = pytest.mark.gpu

REC = np.dtype([("s", "<f8"), ("x2", "<f8"), ("h", "<i8"), ("flag", "i1")])  # packed: 25 bytes
assert REC.itemsize == 25
_MIX = np.array([0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9], dtype=np.uint64)


def row_hash(x):
    """An int64 hash of each row's bits."""
    u = np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)
    mult = _MIX[np.arange(u.shape[-1]) % 3]
    with np.errstate(over="ignore"):
        return np.bitwise_xor.reduce(u * mult + np.arange(u.shape[-1], dtype=np.uint64), axis=-1).view(np.int64)


def blob_of(x):
    x = np.asarray(x, dtype=np.float64)
    out = np.empty(x.shape[:-1], dtype=REC)
    out["s"] = x.sum(-1)
    out["x2"] = 2.0 * x[..., 0]
    out["h"] = row_hash(x)
    out["flag"] = (x[..., 0] > 0).astype(np.int8)
    return out


def lp_of(x):
    """A Gaussian of variance ndim per parameter: every move accepts often at ndim 257 too."""
    x = np.asarray(x)
    return -0.5 * np.sum(x**2, axis=-1) / x.shape[-1]


def rows_result(lp, blobs):
    """A vectorised function's result by the reference's rules (ensemble.py:498-547): one ``(lp, blob...)``
    sequence per row -- a structured record's fields, else its array or scalar."""
    if blobs.dtype.names:
        return [(float(v),) + b.item() for v, b in zip(lp, blobs)]
    return [(float(v), b) for v, b in zip(lp, blobs)]


class Rec(object):
    """A vectorised function with blobs that keeps its inputs."""

    def __init__(self, blobs=True):
        self.inputs, self.blobs = [], blobs

    def __call__(self, x):
        self.inputs.append(np.array(x, copy=True))
        return rows_result(lp_of(x), blob_of(x)) if self.blobs else lp_of(x)


def host_fn(blobs=True, rec=None):
    rec = rec or Rec(blobs)
    return models.HostFunction(rec, vectorize=True, blobs_dtype=REC if blobs else None), rec


def _full_cov(D):
    a = np.random.default_rng(D).standard_normal((D, D))
    return 0.01 * (a @ a.T) + 0.1 * np.eye(D)


MOVES = [
    ("stretch", lambda P, D: moves.StretchMove(nsplits=P)),
    ("de", lambda P, D: moves.DEMove(nsplits=P)),
    ("snooker", lambda P, D: moves.DESnookerMove()),
    ("walk", lambda P, D: moves.WalkMove(nsplits=P)),
    ("walk_subset", lambda P, D: moves.WalkMove(s=4, nsplits=P)),
    ("gauss_scalar", lambda P, D: moves.GaussianMove(0.3)),
    ("gauss_diag_random", lambda P, D: moves.GaussianMove(np.linspace(0.1, 0.4, D), mode="random", factor=1.5)),
    ("gauss_sequential", lambda P, D: moves.GaussianMove(np.linspace(0.1, 0.4, D), mode="sequential")),
    ("gauss_full", lambda P, D: moves.GaussianMove(_full_cov(D))),
    ("mh_gauss_mix", lambda P, D: [(moves.StretchMove(nsplits=P), 0.5), (moves.GaussianMove(0.2), 0.5)]),
]


def _torch():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("torch has no CUDA")
    return torch


def _torch_blob_fn(torch, mode="current", sleep=False, strided=False):
    """(lp, blobs) in torch: blobs are float64 [M, 4] = (sum, 2 x0, x0, x_last).  mode "v3" writes on a side
    stream named in a v3 interface; "side" on a side stream with torch's own (v2) interface."""
    stream = torch.cuda.Stream() if mode != "current" else None

    class V3(object):
        def __init__(self, t):
            cai = dict(t.__cuda_array_interface__)
            cai.update(version=3, stream=stream.cuda_stream or 1)
            self.__cuda_array_interface__ = cai
            self.t = t

    def body(rows):
        x = torch.as_tensor(rows, device="cuda")
        lp = (x * x).sum(1) * -0.5
        big = torch.full((x.shape[0], 8 if strided else 4), float("nan"), dtype=torch.float64, device="cuda")
        if sleep:
            torch.cuda._sleep(20_000_000)  # ~10 ms before the final write
        big[:, 0] = x.sum(1)
        big[:, 1] = 2.0 * x[:, 0]
        big[:, 2] = x[:, 0]
        big[:, 3] = x[:, -1]
        b = big[:, :4]
        if mode == "v3":
            return V3(lp * 1.0), V3(b)
        return lp * 1.0, b

    def f(rows):
        if stream is None:
            return body(rows)
        with torch.cuda.stream(stream):
            return body(rows)

    return f


def _torch_blob_ref(x):
    x = np.asarray(x)
    return np.stack([x.sum(-1), 2.0 * x[..., 0], x[..., 0], x[..., -1]], axis=-1)


def _device_fn_numpy():
    """A device-mode function that returns numpy results: the rows are read with torch."""
    torch = _torch()

    def f(rows):
        x = torch.as_tensor(rows, device="cuda").cpu().numpy()
        return lp_of(x), blob_of(x)

    return models.CudaArrayFunction(f, blobs_dtype=REC)


def _torch_pure_fn():
    """Device mode with CUDA-array results: int64 records [M, 4] computed by torch on the device -- the bits of
    x[0], 2 x[0] and x[-1], and a wrapping integer hash of the row -- returned as a view with a strided first
    axis (40-byte rows holding 32-byte records)."""
    torch = _torch()
    mix = {}

    def f(rows):
        x = torch.as_tensor(rows, device="cuda")
        D = x.shape[1]
        if D not in mix:
            mix[D] = torch.as_tensor(_MIX.view(np.int64)[np.arange(D) % 3], device="cuda")
        xi = x.view(torch.int64)
        buf = torch.empty((x.shape[0], 5), dtype=torch.int64, device="cuda")
        buf[:, 0] = xi[:, 0]
        buf[:, 1] = (2.0 * x[:, 0]).view(torch.int64)
        buf[:, 2] = xi[:, -1]
        buf[:, 3] = (xi * mix[D]).sum(1)
        return (x * x).sum(1) * (-0.5 / D), buf[:, :4]

    return models.CudaArrayFunction(f, blobs_dtype=np.int64)


def torch_blob_of(x):
    x = np.ascontiguousarray(x, dtype=np.float64)
    xi = x.view(np.int64)
    mix = _MIX.view(np.int64)[np.arange(x.shape[-1]) % 3]
    with np.errstate(over="ignore"):
        h = (xi * mix).sum(-1)  # wraps, as int64 does on the device: the sum's order does not matter
    return np.stack([xi[..., 0], np.ascontiguousarray(2.0 * x[..., 0]).view(np.int64), xi[..., -1], h], axis=-1)


def _check_pure(s, states, f=blob_of):
    chain, blobs = s.get_chain(), s.get_blobs()
    ref = f(chain)
    assert blobs.dtype == ref.dtype and blobs.shape == ref.shape
    assert blobs.tobytes() == ref.tobytes()
    for st in states:
        assert st.blobs.tobytes() == f(st.coords).tobytes()


# ---- 1. the blob is a pure function of the row -------------------------------------------------------------------
@pytest.mark.parametrize("where", ["host", "device", "torch"])
@pytest.mark.parametrize("D", [1, 33, 257])
@pytest.mark.parametrize("P", [2, 3, 5])
@pytest.mark.parametrize("kind,make", MOVES, ids=[m[0] for m in MOVES])
def test_blobs_follow_their_walker(kind, make, P, D, where):
    if (kind.startswith("gauss") or kind == "snooker") and P != 2:
        pytest.skip("no split count to vary")
    if kind == "walk_subset" and D > 64:
        pytest.skip("WalkMove helper subsets are limited to ndim <= 64")
    N = max(2 * D + 1, 41) | 1  # odd
    fn = {"host": lambda: host_fn()[0], "device": _device_fn_numpy, "torch": _torch_pure_fn}[where]()
    s = emcee_b200.EnsembleSampler(N, D, fn, moves=make(P, D), seed=0xB10B + D + P)
    p0 = np.random.default_rng(D).standard_normal((N, D))
    states = [emcee_b200.State(st, copy=True) for st in s.sample(p0, iterations=3, skip_initial_state_check=True)]
    last = s.run_mcmc(states[-1], 3)  # the bulk path into the same backend, from a State that carries blobs
    states.append(last)
    _check_pure(s, states, torch_blob_of if where == "torch" else blob_of)
    assert s.backend.iteration == 6 and np.any(s.backend.accepted > 0)


@pytest.mark.parametrize("kind,make", MOVES[:6], ids=[m[0] for m in MOVES[:6]])
def test_walkers_from_minus_inf_take_every_proposal(kind, make):
    N, D = 41, 4
    p0 = np.random.default_rng(2).standard_normal((N, D))
    s = emcee_b200.EnsembleSampler(N, D, host_fn()[0], moves=make(2, D), seed=5)
    start = emcee_b200.State(p0, log_prob=np.full(N, -np.inf), blobs=blob_of(p0))
    last = s.run_mcmc(start, 1, skip_initial_state_check=True)
    assert np.all(s.backend.accepted == 1)
    assert last.blobs.tobytes() == blob_of(last.coords).tobytes()


# ---- 2. blobs change nothing else -------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,make", MOVES, ids=[m[0] for m in MOVES])
def test_twin_runs_with_and_without_blobs(kind, make):
    N, D = 37, 5
    p0 = np.random.default_rng(3).standard_normal((N, D))
    runs = []
    for blobs in (True, False):
        fn, rec = host_fn(blobs)
        s = emcee_b200.EnsembleSampler(N, D, fn, moves=make(3, D), seed=0x7A1)
        s.run_mcmc(p0, 8, skip_initial_state_check=True)
        runs.append((s, rec))
    (a, ra), (b, rb) = runs
    assert np.array_equal(a.get_chain(), b.get_chain()) and np.array_equal(a.get_log_prob(), b.get_log_prob())
    assert np.array_equal(a.backend.accepted, b.backend.accepted)
    assert len(ra.inputs) == len(rb.inputs) and all(np.array_equal(x, y) for x, y in zip(ra.inputs, rb.inputs))
    assert a._engine.get_rng() == b._engine.get_rng() and b.get_blobs() is None


# ---- 3. record sizes: every copy width ---------------------------------------------------------------------------
# (dtype of one element, record shape): 1, 2, 3, 4, 6, 8, 12, 16, 24, 1000 and 25 (packed structured) bytes --
# the 16-, 8-, 4-, 2- and 1-byte copies of blob_select_kernel
SIZES = [("b1", ()), ("i2", ()), ("i1", (3,)), ("f4", ()), ("i2", (3,)), ("f8", ()), ("f4", (3,)), ("f8", (2,)),
         ("f8", (3,)), ("u1", (1000,)), ("i1", ()), (REC, ())]


def _records(x, base, shape):
    """Records of dtype `base` and shape `shape` whose bytes are a function of the row."""
    base = np.dtype(base)
    h = row_hash(x).view(np.uint64)
    n = base.itemsize * (int(np.prod(shape)) if shape else 1)
    raw = np.empty(x.shape[:-1] + (n,), dtype=np.uint8)
    for j in range(n):
        raw[..., j] = ((h >> np.uint64(8 * (j % 8))) + np.uint64(j // 8)).astype(np.uint8)
    if base.kind == "b":
        raw &= 1
    # floats stay finite (a NaN may lose its payload bits on the way through Python floats)
    fields = [(t, o) for t, o in (v[:2] for v in base.fields.values())] if base.names else [(base, 0)]
    for t, o in fields:
        if t.kind == "f":
            raw[..., o + t.itemsize - 1 :: base.itemsize] &= 0x3F
    out = raw.view(base)
    return out[..., 0] if base.names else out.reshape(x.shape[:-1] + shape)


@pytest.mark.parametrize("base,shape", SIZES, ids=["%s%s" % (np.dtype(b).itemsize, s) for b, s in SIZES])
def test_record_sizes(base, shape):
    def f(x):
        return rows_result(lp_of(x), _records(x, base, shape))

    N, D = 33, 3
    s = emcee_b200.EnsembleSampler(N, D, models.HostFunction(f, vectorize=True, blobs_dtype=base), seed=11)
    s.run_mcmc(np.random.default_rng(4).standard_normal((N, D)), 5, skip_initial_state_check=True)
    blobs = s.get_blobs()
    assert blobs.dtype == np.dtype(base) and blobs.shape == (5, N) + shape
    assert blobs.tobytes() == np.ascontiguousarray(_records(s.get_chain(), base, shape)).tobytes()


def test_subarray_dtype_device_mode():
    torch = _torch()
    dt = np.dtype(("f4", (3,)))  # 12-byte records

    def f(rows):
        x = torch.as_tensor(rows, device="cuda")
        return (x * x).sum(1) * -0.5, x[:, :3].to(torch.float32)

    N, D = 33, 5
    s = emcee_b200.EnsembleSampler(N, D, models.CudaArrayFunction(f, blobs_dtype=dt), seed=12)
    s.run_mcmc(np.random.default_rng(5).standard_normal((N, D)), 5, skip_initial_state_check=True)
    blobs = s.get_blobs()
    assert blobs.dtype == np.float32 and blobs.shape == (5, N, 3)
    assert np.array_equal(blobs, s.get_chain()[..., :3].astype(np.float32))


# ---- 4. the reference's flows and the edges ----------------------------------------------------------------------
class Variable(object):
    """The reference's VariableLogProb (tests/unit/test_blobs.py): blobs of length i."""

    def __init__(self):
        self.i = 3

    def __call__(self, x):
        return 0.0, np.zeros(self.i)


def test_blob_mismatch():
    np.random.seed(42)
    model = Variable()
    coords = np.random.randn(32, 3)
    s = emcee_b200.EnsembleSampler(32, 3, models.HostFunction(model, blobs_dtype=float), seed=1)
    model.i += 1
    s.run_mcmc(coords, 1)
    assert s.get_blobs().shape == (1, 32, 4)
    model.i += 1
    with pytest.raises(ValueError):
        s.run_mcmc(coords, 1)
    # within a run: the layout is fixed by the initial evaluation
    m2 = Variable()
    batches = {"n": 0}

    def bump(xs):
        batches["n"] += 1
        if batches["n"] == 2:  # the first half-step's records are one longer than the state's
            m2.i += 1
        return [m2(x) for x in xs]

    s3 = emcee_b200.EnsembleSampler(32, 3, models.HostFunction(bump, vectorize=True, blobs_dtype=float), seed=1)
    with pytest.raises(ValueError, match="shape"):
        s3.run_mcmc(coords, 2)
    assert s3.backend.iteration == 0


def test_function_stops_returning_blobs_and_log_prob_without_blobs():
    calls = {"n": 0}

    def f(x):
        calls["n"] += 1
        return rows_result(lp_of(x), blob_of(x)) if calls["n"] < 3 else lp_of(x)

    p0 = np.random.default_rng(5).standard_normal((32, 4))
    s = emcee_b200.EnsembleSampler(32, 4, models.HostFunction(f, vectorize=True, blobs_dtype=REC), seed=2)
    with pytest.raises(ValueError, match="no blobs"):
        s.run_mcmc(p0, 3, skip_initial_state_check=True)
    assert s.backend.iteration == 0 and s._engine.get_rng()[1] == 0  # stopped inside step 0
    fn = host_fn()[0]
    s = emcee_b200.EnsembleSampler(32, 4, fn, seed=2)
    with pytest.raises(ValueError, match="If you start sampling with a given log_prob"):
        s.run_mcmc(emcee_b200.State(p0, log_prob=lp_of(p0)), 2, skip_initial_state_check=True)
    coords, lp = s._engine.get_state()
    assert np.array_equal(coords, p0) and np.array_equal(lp, lp_of(p0))  # refused before any update


def test_state_blobs_checked_before_anything_runs():
    p0 = np.random.default_rng(5).standard_normal((32, 4))
    fn, rec = host_fn()
    s = emcee_b200.EnsembleSampler(32, 4, fn, seed=2)
    with pytest.raises(NotImplementedError, match="fixed-width"):
        s.run_mcmc(emcee_b200.State(p0, log_prob=lp_of(p0), blobs=np.array([object()] * 32)), 2,
                   skip_initial_state_check=True)
    with pytest.raises(ValueError, match="declares"):
        s.run_mcmc(emcee_b200.State(p0, log_prob=lp_of(p0), blobs=np.zeros(32)), 2, skip_initial_state_check=True)
    assert rec.inputs == [] and not s.backend.has_blobs() and s.backend.iteration == 0
    # the backend was left untouched, so the right blobs still run
    s.run_mcmc(emcee_b200.State(p0, log_prob=lp_of(p0), blobs=blob_of(p0)), 2, skip_initial_state_check=True)
    assert s.get_blobs().tobytes() == blob_of(s.get_chain()).tobytes()


def test_device_backend_refused():
    with pytest.raises(NotImplementedError, match=r"Backend\(\)"):
        emcee_b200.EnsembleSampler(32, 4, host_fn()[0], backend=emcee_b200.DeviceBackend())
    s = emcee_b200.EnsembleSampler(32, 4, host_fn()[0], seed=1)
    s.backend = emcee_b200.DeviceBackend()
    s.backend.reset(32, 4)
    with pytest.raises(NotImplementedError, match=r"Backend\(\)"):
        s.run_mcmc(np.random.default_rng(0).standard_normal((32, 4)), 1, skip_initial_state_check=True)


def _p0():
    return np.random.default_rng(6).standard_normal((40, 4))


def _blob_sampler(fn=None, **kw):
    return emcee_b200.EnsembleSampler(40, 4, fn or host_fn()[0], moves=moves.StretchMove(randomize_split=False),
                                      seed=0xE1, **kw)


@pytest.mark.parametrize("how", ["thin_by", "thin", "store_false", "iterations0", "sample_thin_by"])
def test_storage_paths(how):
    ref = _blob_sampler()
    ref.run_mcmc(_p0(), 12, skip_initial_state_check=True)
    chain, blobs = ref.get_chain(), ref.get_blobs()
    assert blobs.tobytes() == blob_of(chain).tobytes()
    s = _blob_sampler()
    if how == "thin_by":
        s.run_mcmc(_p0(), 4, thin_by=3, skip_initial_state_check=True)
        assert s.get_blobs().tobytes() == blobs[2::3].tobytes()
    elif how == "sample_thin_by":
        for st in s.sample(_p0(), iterations=4, thin_by=3, skip_initial_state_check=True):
            assert st.blobs.tobytes() == blob_of(st.coords).tobytes()
        assert s.get_blobs().tobytes() == blobs[2::3].tobytes()
    elif how == "thin":
        s.run_mcmc(_p0(), 12, thin=3, skip_initial_state_check=True)
        assert s.get_blobs().tobytes() == blobs[2::3].tobytes()
    elif how == "store_false":
        last = s.run_mcmc(_p0(), 12, store=False, skip_initial_state_check=True)
        assert last.blobs.tobytes() == blobs[-1].tobytes()
    else:
        assert s.run_mcmc(_p0(), 0, skip_initial_state_check=True) is None
        last = s.run_mcmc(_p0(), 12, skip_initial_state_check=True)
        assert s.get_blobs().tobytes() == blobs.tobytes() and last.blobs.tobytes() == blobs[-1].tobytes()


class UserError(Exception):
    pass


@pytest.mark.parametrize("path", ["run_mcmc", "sample"])
def test_user_exception_then_resume(path):
    k, j, n = 3, 1, 7
    calls = {"n": 0}

    def f(x):
        calls["n"] += 1
        if calls["n"] == 1 + 1 + 2 * k + j:
            raise UserError("user failure")
        return rows_result(lp_of(x), blob_of(x))

    s = _blob_sampler(models.HostFunction(f, vectorize=True, blobs_dtype=REC))
    with pytest.raises(UserError):
        if path == "run_mcmc":
            s.run_mcmc(_p0(), n, skip_initial_state_check=True)
        else:
            for _ in s.sample(_p0(), iterations=n, skip_initial_state_check=True):
                pass
    tw = _blob_sampler()
    tw.run_mcmc(_p0(), n, skip_initial_state_check=True)
    assert s.backend.iteration == k
    assert s.get_blobs().tobytes() == tw.get_blobs()[:k].tobytes()
    last = s.get_last_sample()
    assert last.blobs.tobytes() == tw.get_blobs()[k - 1].tobytes()
    s.run_mcmc(last, n - k)
    assert np.array_equal(s.get_chain(), tw.get_chain()) and np.array_equal(s.get_log_prob(), tw.get_log_prob())
    assert s.get_blobs().tobytes() == tw.get_blobs().tobytes()


def test_pickling_continues_identically():
    a = _blob_sampler()
    a.run_mcmc(_p0(), 4, skip_initial_state_check=True)
    b = pickle.loads(pickle.dumps(a))
    assert b.get_blobs().tobytes() == a.get_blobs().tobytes()
    a.run_mcmc(None, 5)
    b.run_mcmc(None, 5)
    assert np.array_equal(a.get_chain(), b.get_chain()) and a.get_blobs().tobytes() == b.get_blobs().tobytes()
    bk = pickle.loads(pickle.dumps(a.backend))
    assert bk.get_blobs().tobytes() == a.get_blobs().tobytes()


def test_compute_log_prob():
    s = _blob_sampler()
    x = np.random.default_rng(7).standard_normal((3, 5, 4))
    lp, blobs = s.compute_log_prob(x)  # before any state: any layout
    assert np.array_equal(lp, lp_of(x)) and blobs.shape == (3, 5) and blobs.tobytes() == blob_of(x).tobytes()
    s.run_mcmc(_p0(), 2, skip_initial_state_check=True)
    lp, blobs = s.compute_log_prob(x[0])
    assert blobs.tobytes() == blob_of(x[0]).tobytes()
    with pytest.raises(ValueError, match="infinite"):
        y = x.copy()
        y[0, 0, 0] = np.inf
        s.compute_log_prob(y)


# ---- 5. torch CUDA-array blobs ----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,strided", [("v3", False), ("side", False), ("current", True)])
def test_torch_blobs(mode, strided):
    torch = _torch()
    N, D = 64, 7
    p0 = np.random.default_rng(8).standard_normal((N, D))
    mv = [(moves.StretchMove(), 0.5), (moves.DEMove(), 0.3), (moves.WalkMove(), 0.2)]
    s = emcee_b200.EnsembleSampler(
        N, D, models.CudaArrayFunction(_torch_blob_fn(torch, mode, sleep=True, strided=strided), blobs_dtype="f8"),
        moves=mv, seed=11)
    s.run_mcmc(p0, 8, skip_initial_state_check=True)
    assert s._engine.last_kernel_variant().endswith("where=device")
    blobs, chain = s.get_blobs(), s.get_chain()
    assert blobs.shape == (8, N, 4)
    np.testing.assert_array_equal(blobs[..., 1:], _torch_blob_ref(chain)[..., 1:])
    np.testing.assert_allclose(blobs[..., 0], chain.sum(-1), rtol=1e-13, atol=1e-13)  # torch's summation order


# ---- 6. at scale --------------------------------------------------------------------------------------------------
def test_at_scale_device_mode():
    torch = _torch()
    N, D = 65536, 128

    def f(rows):
        x = torch.as_tensor(rows, device="cuda")
        lp = (x * x).sum(1) * -0.5
        b = torch.stack([x[:, 0], x[:, -1]], dim=1)  # 16-byte records
        return lp, b

    s = emcee_b200.EnsembleSampler(N, D, models.CudaArrayFunction(f, blobs_dtype="f8"), seed=0x5CA1E)
    p0 = np.random.default_rng(9).standard_normal((N, D))
    s.run_mcmc(p0, 3, thin_by=10, skip_initial_state_check=True)  # 30 steps, 3 stored
    chain, blobs = s.get_chain(), s.get_blobs()
    assert blobs.shape == (3, N, 2)
    pick = np.random.default_rng(10).choice(N, 2048, replace=False)
    assert np.array_equal(blobs[:, pick, 0], chain[:, pick, 0]) and np.array_equal(blobs[:, pick, 1], chain[:, pick, -1])
    assert s.backend.accepted.mean() > 0.1  # the accept masks of the three stored steps: selection was exercised
