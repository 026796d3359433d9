"""Host-side mirror of the reference's operator interface for the AGD hot path, over the C-ABI.

Names, argument meaning and error behaviour follow
/root/reference/src/main/scala/org/apache/spark/mllib/optimization/AcceleratedGradientDescent.scala
(class AcceleratedGradientDescent :41-144, object AcceleratedGradientDescent.run :177-338) and the
spark-mllib 1.3.0 plug-in types it is given (Gradient / Updater).  The Scala/JVM facade a Spark
maintainer would compile is shipped as source under jvm/ (no JVM in this image); this module is the
executable mirror used by the tests and the benchmark.

  sc = Context(devices=[0])                      # ~ SparkContext: which GPUs, which communicator
  data = sc.parallelize(labels, X).cache()       # ~ RDD[(Double, Vector)] pinned in HBM (Suite.scala:51)
  w, loss = AcceleratedGradientDescent.run(data, LogisticGradient(), SimpleUpdater(), 1e-12, 10, 0.0,
                                           w0, 1.0, float("inf"), 0.5, 0.9, True)      # Suite.scala:62-74
  w = AcceleratedGradientDescent(LogisticGradient(), SquaredL2Updater()).setRegParam(0.2).optimize(data, w0)
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

from . import _native as N


# --------------------------------------------------------------------------- plug-in types
class Gradient:
    """org.apache.spark.mllib.optimization.Gradient [mllib-1.3.0]: closed set of built-ins."""
    kind: int = -1


class LogisticGradient(Gradient):
    kind = N.GRAD_LOGISTIC

    def __init__(self, numClasses: int = 2):
        if numClasses != 2:  # the reference only ever builds the binary form (Suite.scala:39,251)
            raise NotImplementedError("multinomial LogisticGradient is outside the reference's AGD path")


class LeastSquaresGradient(Gradient):
    """1.3.0 definition: loss diff^2, gradient 2*diff*x.  half=True selects the Spark>=1.4 definition."""

    def __init__(self, half: bool = False):
        self.kind = N.GRAD_LEAST_SQUARES_HALF if half else N.GRAD_LEAST_SQUARES


class HingeGradient(Gradient):
    kind = N.GRAD_HINGE


class Updater:
    """org.apache.spark.mllib.optimization.Updater [mllib-1.3.0]: closed set of built-ins."""
    kind: int = -1


class SimpleUpdater(Updater):
    kind = N.UPD_SIMPLE


class SquaredL2Updater(Updater):
    kind = N.UPD_SQUARED_L2


class L1Updater(Updater):
    kind = N.UPD_L1


def _grad_kind(g) -> int:
    if not isinstance(g, Gradient) or g.kind < 0:
        # the JVM facade throws UnsupportedOperationException here: there is no CPU fallback
        raise TypeError(f"unsupported Gradient {type(g).__name__}: only Logistic/LeastSquares/Hinge run on the GPU path")
    return g.kind


def _upd_kind(u) -> int:
    if not isinstance(u, Updater) or u.kind < 0:
        raise TypeError(f"unsupported Updater {type(u).__name__}: only Simple/SquaredL2/L1 run on the GPU path")
    return u.kind


_DT = {np.dtype(np.float64): N.F64, np.dtype(np.float32): N.F32}
_STORE = {"f32": N.F32, "f64": N.F64, "bf16": N.BF16, N.F32: N.F32, N.F64: N.F64, N.BF16: N.BF16}


def bf16_to_f32(raw: np.ndarray) -> np.ndarray:
    """Exact widening of raw bf16 bit patterns (uint16) to float32."""
    return (raw.astype(np.uint32) << 16).view(np.float32)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# --------------------------------------------------------------------------- context + dataset
class Context:
    """Which local GPUs this process drives and how its ranks sit in the world (one rank per GPU).

    devices: local CUDA ordinals.  world_size/first_rank: global layout.  Multi-process worlds
    (world_size > len(devices)) pick how the exchange is SET UP (the per-pass data never touches a library):
      transport="nccl": id_exchange(bytes|None) -> bytes returns rank 0's 128-byte NCCL id on every process
                        (e.g. a torch.distributed broadcast); NCCL ships the CUDA IPC handles and is the fallback;
      transport="ipc":  handle_exchange(bytes) -> bytes returns every process's handle blob concatenated in rank
                        order (an all-gather in the host language); no NCCL anywhere -- also works for several
                        processes sharing one GPU."""

    def __init__(self, devices: Sequence[int] = (0,), world_size: Optional[int] = None, first_rank: int = 0,
                 id_exchange=None, handle_exchange=None, transport: Optional[str] = None):
        self.devices = list(devices)
        self.world_size = len(self.devices) if world_size is None else int(world_size)
        self.first_rank = int(first_rank)
        self.id_exchange = id_exchange
        self.handle_exchange = handle_exchange
        self.transport = transport or ("ipc" if (handle_exchange is not None and id_exchange is None) else "nccl")
        if self.transport not in ("nccl", "ipc"):
            raise ValueError("transport must be 'nccl' or 'ipc'")
        if self.world_size > len(self.devices):
            if self.transport == "nccl" and id_exchange is None:
                raise ValueError("multi-process worlds need id_exchange to ship the NCCL unique id")
            if self.transport == "ipc" and handle_exchange is None:
                raise ValueError("transport='ipc' needs handle_exchange to ship the CUDA IPC handles")

    @staticmethod
    def from_torch_distributed(local_device: Optional[int] = None, transport: str = "nccl") -> "Context":
        """One process per GPU under torchrun: ranks/ids/handles travel over the existing process group."""
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(), dist.get_world_size()
        dev = torch.cuda.current_device() if local_device is None else local_device

        def exchange(my_id):
            buf = [my_id]
            dist.broadcast_object_list(buf, src=0)
            return buf[0]

        def gather_handles(blob):
            out = [None] * world
            dist.all_gather_object(out, blob)
            return b"".join(out)

        return Context([dev], world_size=world, first_rank=rank, id_exchange=exchange, handle_exchange=gather_handles,
                       transport=transport)

    def _new_handle(self) -> C.c_void_p:
        L = N.lib()
        ids = (C.c_int32 * len(self.devices))(*self.devices)
        h = C.c_void_p()
        N.check(L.agd_create(ids, len(self.devices), C.byref(h)), None)
        if self.world_size > len(self.devices) and self.transport == "ipc":
            N.check(L.agd_comm_init_ipc(h, self.world_size, self.first_rank), h)
        elif self.world_size > len(self.devices):
            my_id = None
            if self.first_rank == 0:
                buf = C.create_string_buffer(128)
                N.check(L.agd_comm_unique_id(buf), None)
                my_id = buf.raw
            the_id = self.id_exchange(my_id)
            N.check(L.agd_comm_init(h, C.c_char_p(the_id), self.world_size, self.first_rank), h)
        return h

    # --- RDD construction (mirrors sc.parallelize(data, numSlices).cache(), Suite.scala:51) ---
    def parallelize(self, labels, X, store: str = "f64") -> "DeviceDataset":
        """Rows of THIS process are split contiguously over its local GPUs."""
        ds = DeviceDataset(self)
        ds.load_dense(labels, X, store=store)
        return ds

    def parallelize_csr(self, labels, rowptr, idx, val, d: int, store: str = "f64") -> "DeviceDataset":
        ds = DeviceDataset(self)
        ds.load_csr(labels, rowptr, idx, val, d, store=store)
        return ds

    def synthetic(self, total_rows: int, d: int, gradient: Gradient, seed: int = 42, store: str = "f32") -> "DeviceDataset":
        """The benchmark workload of SURVEY.md 8(d), generated in place on every GPU rank."""
        ds = DeviceDataset(self)
        N.check(N.lib().agd_generate(ds.h, total_rows, d, _STORE[store], seed, _grad_kind(gradient)), ds.h)
        ds.total_rows = total_rows
        return ds


def _synthetic_csr(ctx, total_rows, d, nnz_per_row, gradient, seed=42, store="f32"):
    ds = DeviceDataset(ctx)
    N.check(N.lib().agd_generate_csr(ds.h, total_rows, d, nnz_per_row, _STORE[store], seed, _grad_kind(gradient)), ds.h)
    ds.total_rows = total_rows
    return ds


Context.synthetic_csr = _synthetic_csr


# Views (randomSplit / sample / kFold): a predicate (seed, lo, hi, complement) keeps row r iff lo <= u(seed, r) < hi on the
# row's own 64-bit Philox draw (include/agd_b200.h, agd_set_row_filter), negated when complemented; a view keeps the rows
# every one of its predicates keeps.  Every rank of a world must select the same rows, so the default seed is fixed, not
# random.
DEFAULT_SPLIT_SEED = 42
MAX_VIEW_PREDICATES = 4


def split_bounds(weights) -> list:
    """RDD.randomSplit's cell bounds: the weights normalised by their sum and accumulated in fp64
    (weights.map(_ / sum).scanLeft(0.0)(_ + _)).  The last bound is 1, so rounding in the sum can leave no row out."""
    w = [float(x) for x in weights]
    if not w:
        raise ValueError("randomSplit needs at least one weight")
    if any(not (x >= 0.0) or x == float("inf") for x in w):
        raise ValueError(f"weights must be finite and nonnegative, got {weights}")
    total = sum(w)
    if not (total > 0.0):
        raise ValueError(f"sum of weights must be positive, got {weights}")
    bounds = [0.0]
    for x in w:
        bounds.append(bounds[-1] + x / total)
    bounds = [min(b, 1.0) for b in bounds]
    bounds[-1] = 1.0
    return bounds


class DeviceDataset:
    """RDD[(Double, Vector)] stand-in: row shards pinned in HBM for the lifetime of the object.

    randomSplit / sample / MLUtils.kFold return views: DeviceDatasets that share this one's shards and handle and select
    rows by a fixed predicate on each row's own random draw, without copying a row.  Every compute call on a view (smooth*,
    evaluate, margins, training) sets the view's filter on the handle for that call only; close() on a view frees nothing.
    The accessors that address PHYSICAL rows -- local_rows, get_rows, get_labels, get_csr_rows, margins_rows -- return the
    parent's rows on a view as well (the view's own rows of them: row_mask; its row count: count()).

    StandardScalerModel.transform and MLUtils.appendBias return views too: features scaled by s and / or a constant 1.0
    appended, computed on the stored rows without rewriting them (agd_set_feature_transform).  `d` reports the transformed
    width; the physical-row accessors still return the stored features.  Transforms and row views compose in either order."""

    _scale = None      # a transformed view: the factor s of every stored feature (None: unscaled) ...
    _bias = False      # ... and whether a constant 1.0 is appended as the last feature

    def __init__(self, ctx: Context):
        self.ctx = ctx
        self.h = ctx._new_handle()
        self.total_rows = 0
        self._xchg_d = 0       # dimension the host-shipped exchange (transport="ipc") was set up for
        self._base = None      # a view: the dataset that owns the shards (kept alive by this reference)
        self._preds = ()       # a view: its predicates (seed, lo, hi, complement)

    def _view(self, pred) -> "DeviceDataset":
        preds = self._preds + ((pred,) if pred is not None else ())
        if len(preds) > MAX_VIEW_PREDICATES:
            raise ValueError(f"a view nests at most {MAX_VIEW_PREDICATES} predicates (randomSplit / sample / kFold levels)")
        if pred is not None:
            seed, lo, hi, comp = pred
            if not (0.0 <= lo <= hi <= 1.0):
                raise ValueError(f"bounds must satisfy 0 <= lo <= hi <= 1, got [{lo}, {hi})")
        v = object.__new__(DeviceDataset)
        v.ctx = self.ctx
        v._base = self._base if self._base is not None else self
        v.h = v._base.h
        v.total_rows = v._base.total_rows
        v._xchg_d = 0
        v._preds = preds
        v._scale, v._bias = self._scale, self._bias
        return v

    def _transformed(self, scale=None, bias: bool = False) -> "DeviceDataset":
        """A view with the stored features multiplied by `scale` and / or a constant 1.0 appended (MLlib's order: scale,
        then appendBias).  It keeps this dataset's rows; a row view of it keeps the transform."""
        if self._bias:
            raise ValueError("this view already ends in the appended bias column: appendBias comes last, after any scaling")
        if scale is not None and self._scale is not None:
            raise ValueError("this view is already scaled; fit and apply one StandardScalerModel")
        v = self._view(None)
        if scale is not None:
            scale = np.array(scale, dtype=np.float64, copy=True)
            if scale.ndim != 1 or scale.shape[0] != self._phys_d:
                raise ValueError(f"scale has size {scale.shape}, data has {self._phys_d} features")
            if not np.all(np.isfinite(scale)):
                raise ValueError("scale factors must be finite")
            scale.setflags(write=False)
            v._scale = scale
        v._bias = self._bias or bool(bias)
        return v

    def _physical_model(self, w, intercept: float):
        """A model of this view's features as a model of the stored ones (what agd_margins / agd_evaluate score)."""
        return physical_model(w, intercept, self._scale, self._bias)

    @property
    def is_view(self) -> bool:
        return self._base is not None

    def _filtered(self):
        """Context manager: the view's filter and feature transform are on the handle for the duration of one call, and
        cleared afterwards, also on error (the parent and sibling views never see them).  A dataset that is not a view leaves
        the handle alone."""
        ds = self
        transformed = ds._scale is not None or ds._bias

        class _F:
            def __enter__(self_):
                try:
                    if ds._preds:
                        n = len(ds._preds)
                        seeds = np.array([p[0] for p in ds._preds], dtype=np.uint64)
                        lo = np.array([p[1] for p in ds._preds], dtype=np.float64)
                        hi = np.array([p[2] for p in ds._preds], dtype=np.float64)
                        comp = np.array([1 if p[3] else 0 for p in ds._preds], dtype=np.int32)
                        N.check(N.lib().agd_set_row_filter(ds.h, n, _ptr(seeds), _ptr(lo), _ptr(hi), _ptr(comp)), ds.h)
                    if transformed:
                        N.check(N.lib().agd_set_feature_transform(ds.h, _ptr(ds._scale), int(ds._bias)), ds.h)
                except BaseException:
                    self_.__exit__()
                    raise

            def __exit__(self_, *exc):
                if transformed:
                    N.check(N.lib().agd_set_feature_transform(ds.h, None, 0), ds.h)
                if ds._preds:
                    N.check(N.lib().agd_set_row_filter(ds.h, 0, None, None, None, None), ds.h)
                return False

        return _F()

    # --- views (RDD.randomSplit, RDD.sample, MLUtils.kFold) ---
    def randomSplit(self, weights, seed: int = DEFAULT_SPLIT_SEED) -> list:
        """RDD.randomSplit(weights, seed): disjoint views that cover every row; split k keeps the rows whose draw lies in
        [c_k, c_{k+1}) of the normalised cumulative weights (split_bounds)."""
        b = split_bounds(weights)
        return [self._view((int(seed), b[k], b[k + 1], False)) for k in range(len(b) - 1)]

    def sample(self, withReplacement: bool, fraction: float, seed: int = DEFAULT_SPLIT_SEED) -> "DeviceDataset":
        """RDD.sample(False, fraction, seed): a Bernoulli view keeping the rows whose draw lies in [0, fraction)."""
        if withReplacement:
            raise NotImplementedError("sample(withReplacement=True) needs per-row multiplicities; only Bernoulli views exist")
        fraction = float(fraction)
        if not (0.0 <= fraction <= 1.0):
            raise ValueError(f"fraction must be in [0, 1] without replacement, got {fraction}")
        return self._view((int(seed), 0.0, fraction, False))

    def count(self) -> int:
        """Rows of this dataset (or view) over every shard of the world (collective: one evaluation sweep)."""
        return int(self.evaluate(LeastSquaresGradient(), np.zeros(self.d)).count)

    def row_mask(self, dev: int, row0: int, rows: int) -> np.ndarray:
        """Which physical rows [row0, row0 + rows) of local device `dev`'s shard this view keeps (bool; rank-local)."""
        out = np.empty(max(int(rows), 0), dtype=np.uint8)
        with self._filtered():
            N.check(N.lib().agd_row_filter_mask(self.h, dev, int(row0), int(rows), _ptr(out) if rows > 0 else None), self.h)
        return out.astype(bool)

    def _ensure_exchange(self):
        """transport="ipc": ship the CUDA IPC handles of the exchange buffers once per loaded dimension (collective:
        every process reaches this from the same compute call)."""
        if self._base is not None:
            return self._base._ensure_exchange()
        c = self.ctx
        if c.transport != "ipc" or c.world_size <= len(c.devices) or self._xchg_d == self.d:
            return
        L = N.lib()
        cap = len(c.devices) * N.XCHG_HANDLE_BYTES
        blob = C.create_string_buffer(cap)
        n = C.c_int64()
        N.check(L.agd_xchg_export(self.h, blob, cap, C.byref(n)), self.h)
        everyone = c.handle_exchange(blob.raw[:n.value])
        N.check(L.agd_xchg_import(self.h, C.c_char_p(everyone), len(everyone)), self.h)
        self._xchg_d = self.d

    def cache(self) -> "DeviceDataset":  # shards are always resident; kept for call-site parity
        return self

    def unpersist(self) -> "DeviceDataset":
        """Drops every shard but keeps the context (devices, communicator) for the next load."""
        self._no_view("unpersist")
        N.check(N.lib().agd_clear(self.h), self.h)
        self.total_rows = 0
        self._xchg_d = 0
        return self

    def _no_view(self, what: str):
        if self._base is not None:
            raise ValueError(f"{what} changes the shards; a view shares its parent's and cannot")

    def load_dense(self, labels, X, store: str = "f64"):
        self._no_view("load_dense")
        labels = np.ascontiguousarray(labels, dtype=np.float64)
        X = np.asarray(X)
        if X.dtype not in _DT:
            X = X.astype(np.float64)
        if X.ndim != 2 or X.shape[0] != labels.shape[0]:
            raise ValueError("X must be (rows, d) with one label per row")
        if not X.flags.c_contiguous:
            X = np.ascontiguousarray(X)
        n, d = X.shape
        nd = len(self.ctx.devices)
        L = N.lib()
        for i in range(nd):
            lo, hi = (i * n) // nd, ((i + 1) * n) // nd
            xs, ls = X[lo:hi], labels[lo:hi]
            N.check(L.agd_load_dense(self.h, i, _ptr(xs) if hi > lo else None, _DT[X.dtype],
                                     _ptr(ls) if hi > lo else None, hi - lo, d, d, _STORE[store]), self.h)
        self.total_rows += n

    def load_csr(self, labels, rowptr, idx, val, d: int, store: str = "f64"):
        self._no_view("load_csr")
        labels = np.ascontiguousarray(labels, dtype=np.float64)
        rowptr = np.ascontiguousarray(rowptr, dtype=np.int64)
        idx = np.ascontiguousarray(idx, dtype=np.int32)
        val = np.ascontiguousarray(val)
        if val.dtype not in _DT:
            val = val.astype(np.float64)
        n = labels.shape[0]
        nd = len(self.ctx.devices)
        L = N.lib()
        for i in range(nd):
            lo, hi = (i * n) // nd, ((i + 1) * n) // nd
            rp = np.ascontiguousarray(rowptr[lo:hi + 1] - rowptr[lo])
            a, b = int(rowptr[lo]), int(rowptr[hi])
            N.check(L.agd_load_csr(self.h, i, _ptr(rp), _ptr(idx[a:b]), _ptr(val[a:b]), _DT[val.dtype],
                                   _ptr(labels[lo:hi]), hi - lo, d, _STORE[store]), self.h)
        self.total_rows += n

    @property
    def _phys_d(self) -> int:
        """Features as stored (what the physical-row accessors return)."""
        return int(N.lib().agd_dim(self.h))

    @property
    def d(self) -> int:
        """Features of this dataset: the stored ones, plus the appended bias column on a view that has one."""
        return self._phys_d + (1 if self._bias else 0)

    def local_rows(self, dev: int = 0) -> int:
        """Physical rows of local device `dev`'s shard (on a view too: the parent's)."""
        return int(N.lib().agd_rows(self.h, dev))

    def get_rows(self, dev: int, row0: int, rows: int, dtype=np.float32):
        """Physical rows as stored (dtype must match the storage: float32, float64, or uint16 for raw bf16); on a view, the
        parent's rows [row0, row0 + rows) -- select the view's with row_mask(dev, row0, rows).  A transformed view returns
        the stored features too (neither scaled nor with the bias column)."""
        X = np.empty((rows, self._phys_d), dtype=dtype)
        y = np.empty(rows, dtype=np.float64)
        N.check(N.lib().agd_get_rows(self.h, dev, row0, rows, _ptr(X), _ptr(y)), self.h)
        return X, y

    def get_labels(self, dev: int, row0: int, rows: int) -> np.ndarray:
        """Labels of physical rows [row0, row0 + rows) (on a view too, as get_rows)."""
        y = np.empty(rows, dtype=np.float64)
        N.check(N.lib().agd_get_rows(self.h, dev, row0, rows, None, _ptr(y)), self.h)
        return y

    def kernel_name(self, dev: int = 0) -> str:
        """The gradient kernel this shard dispatches to (for reports)."""
        return (N.lib().agd_kernel_name(self.h, dev) or b"").decode()

    def get_csr_rows(self, dev: int, row0: int, rows: int, nnz_capacity: int, dtype=np.float32):
        """Physical CSR rows [row0, row0 + rows) (on a view too, as get_rows)."""
        rowptr = np.empty(rows + 1, dtype=np.int64)
        idx = np.empty(nnz_capacity, dtype=np.int32)
        val = np.empty(nnz_capacity, dtype=dtype)
        y = np.empty(rows, dtype=np.float64)
        N.check(N.lib().agd_get_csr_rows(self.h, dev, row0, rows, _ptr(rowptr), _ptr(idx), _ptr(val), nnz_capacity,
                                         _ptr(y)), self.h)
        n = int(rowptr[-1])
        return rowptr, idx[:n], val[:n], y

    def set_option(self, key: str, value) -> None:
        N.check(N.lib().agd_set_option(self.h, key.encode(), str(value).encode()), self.h)

    # plug-in granularity entry points
    def smooth(self, gradient: Gradient, w):
        """applySmooth (AGD.scala:192-208) with host buffers: (loss/count, grad/count, count)."""
        w = np.ascontiguousarray(w, dtype=np.float64)
        if w.shape[0] != self.d:
            raise ValueError("weights have the wrong dimension")
        g = np.empty(self.d, dtype=np.float64)
        loss, cnt = C.c_double(), C.c_int64()
        self._ensure_exchange()
        with self._filtered():
            N.check(N.lib().agd_smooth(self.h, _grad_kind(gradient), _ptr(w), C.byref(loss), _ptr(g), C.byref(cnt)), self.h)
        return loss.value, g, cnt.value

    def smooth_pair(self, gradient: Gradient, w, w2):
        """applySmooth at w plus the loss at w2 from ONE sweep over the shards (the fused form of AGD.scala:250 + :304):
        (loss/count, grad/count, count, loss2/count)."""
        w = np.ascontiguousarray(w, dtype=np.float64)
        w2 = np.ascontiguousarray(w2, dtype=np.float64)
        if w.shape[0] != self.d or w2.shape[0] != self.d:
            raise ValueError("weights have the wrong dimension")
        g = np.empty(self.d, dtype=np.float64)
        loss, loss2, cnt = C.c_double(), C.c_double(), C.c_int64()
        self._ensure_exchange()
        with self._filtered():
            N.check(N.lib().agd_smooth_pair(self.h, _grad_kind(gradient), _ptr(w), _ptr(w2), C.byref(loss), _ptr(g),
                                            C.byref(cnt), C.byref(loss2)), self.h)
        return loss.value, g, cnt.value, loss2.value

    def smooth_two(self, gradient: Gradient, w, w2):
        """Two complete applySmooth evaluations from ONE sweep over the shards: (loss, grad, count, loss2, grad2)."""
        w = np.ascontiguousarray(w, dtype=np.float64)
        w2 = np.ascontiguousarray(w2, dtype=np.float64)
        if w.shape[0] != self.d or w2.shape[0] != self.d:
            raise ValueError("weights have the wrong dimension")
        g, g2 = np.empty(self.d, dtype=np.float64), np.empty(self.d, dtype=np.float64)
        loss, loss2, cnt = C.c_double(), C.c_double(), C.c_int64()
        self._ensure_exchange()
        with self._filtered():
            N.check(N.lib().agd_smooth_two(self.h, _grad_kind(gradient), _ptr(w), _ptr(w2), C.byref(loss), _ptr(g),
                                           C.byref(cnt), C.byref(loss2), _ptr(g2)), self.h)
        return loss.value, g, cnt.value, loss2.value, g2

    # scoring the resident shards (no host copy of X)
    def _weights(self, w) -> np.ndarray:
        w = np.ascontiguousarray(w, dtype=np.float64)
        if w.ndim != 1 or w.shape[0] != self.d:
            raise ValueError(f"weights have size {w.shape}, data has {self.d} features")
        return w

    def margins_rows(self, dev: int, row0: int, rows: int, w, intercept: float = 0.0) -> np.ndarray:
        """x_i . w + intercept (fp64) of physical rows [row0, row0 + rows) of local device `dev`'s shard (not collective; on a
        view too, see margins for the view's rows).  On a transformed view x_i is the transformed row."""
        w, intercept = self._physical_model(self._weights(w), intercept)
        out = np.empty(max(int(rows), 0), dtype=np.float64)
        N.check(N.lib().agd_margins(self.h, dev, _ptr(w), float(intercept), int(row0), int(rows), _ptr(out)), self.h)
        return out

    def margins(self, w, intercept: float = 0.0) -> np.ndarray:
        """x_i . w + intercept (fp64) of this process's rows, across its local devices in load order (not collective); on a
        view, of the view's rows only, in the same order."""
        parts = []
        for i in range(len(self.ctx.devices)):
            m = self.margins_rows(i, 0, self.local_rows(i), w, intercept)
            parts.append(m[self.row_mask(i, 0, m.shape[0])] if self._preds else m)
        return np.concatenate(parts)

    def evaluate(self, gradient: Gradient, w, intercept: float = 0.0, threshold: float = 0.5) -> "Evaluation":
        """Loss, confusion counts and error moments of the model (w, intercept) over every shard of the world, from one
        read of X (collective: every rank calls it; every rank gets the same bits)."""
        w, intercept = self._physical_model(self._weights(w), intercept)
        sums = np.empty(N.EVAL_N, dtype=np.float64)
        self._ensure_exchange()
        with self._filtered():
            N.check(N.lib().agd_evaluate(self.h, _grad_kind(gradient), _ptr(w), float(intercept), float(threshold),
                                         _ptr(sums)), self.h)
        return Evaluation.from_sums(sums)

    def binary_curve(self, w, intercept: float = 0.0, curve: bool = True):
        """The ranking curve of the model (w, intercept) over every shard of the world (agd_binary_curve; collective: every
        rank calls it, every rank gets the same bits): (summary, margins, tp, fp) with summary the AGD_BIN_N doubles [P, N,
        NaN margins, areaUnderROC, areaUnderPR] and, with `curve`, the distinct margins in descending order and the cumulative
        true / false positive counts down to each (None otherwise).  The curve costs a second call of the same kind (the
        first one tells every rank its length)."""
        w, intercept = self._physical_model(self._weights(w), intercept)
        L = N.lib()
        out = np.empty(N.BIN_N, dtype=np.float64)
        k = C.c_int64()
        self._ensure_exchange()
        with self._filtered():
            N.check(L.agd_binary_curve(self.h, _ptr(w), float(intercept), 0, None, None, None, C.byref(k), _ptr(out)), self.h)
            if not curve:
                return out, None, None, None
            n = int(k.value)
            m, tp, fp = np.empty(n), np.empty(n, dtype=np.int64), np.empty(n, dtype=np.int64)
            N.check(L.agd_binary_curve(self.h, _ptr(w), float(intercept), n, _ptr(m) if n else None, _ptr(tp) if n else None,
                                       _ptr(fp) if n else None, C.byref(k), _ptr(out)), self.h)
        return out, m, tp, fp

    def gramian(self, centered: bool):
        """The augmented cross-product matrix of the stored features over every shard of the world (agd_gramian; collective:
        every rank calls it, every rank gets the same bits): (count, A) with A the (d + 1) x (d + 1) matrix [sum z z^T, sum z;
        sum z^T, count], z = x, or x - mu with mu = fl(sum x / count) when `centered`.  On a transformed view these are the
        stored features' sums (linalg.augmented_transformed maps them)."""
        d = self._phys_d
        out = np.empty((d + 1, d + 1), dtype=np.float64) if d <= N.GRAMIAN_MAX_DIM else np.empty(0)   # larger: the call fails
        count = C.c_double()
        self._ensure_exchange()
        with self._filtered():
            N.check(N.lib().agd_gramian(self.h, 1 if centered else 0, C.byref(count), _ptr(out)), self.h)
        return count.value, out

    def project(self, B, offset=None, store: str = "f64") -> "DeviceDataset":
        """RowMatrix.multiply on the device (agd_project): a new dataset whose rows are this dataset's (or view's) rows times B
        ((d, k) array, d = self.d) plus `offset` (k values, None = 0), stored as `store`, each with its label, in physical
        order on the same devices.  A transformed view is folded into B and offset first (physical_projection).  Rank-local,
        but the new dataset is opened on this one's context, so in a multi-process world every rank calls it.  The result owns
        its shards: close() frees them."""
        P, c = physical_projection(B, offset, self._scale, self._bias, self.d)
        out = DeviceDataset(self.ctx)
        try:
            with self._filtered():
                N.check(N.lib().agd_project(self.h, _ptr(P), P.shape[1], _ptr(c), out.h, _STORE[store]), self.h)
        except BaseException:
            out.close()
            raise
        out.total_rows = sum(out.local_rows(i) for i in range(len(self.ctx.devices)))
        return out

    # clustering (agd_kmeans_*): in this dataset's (or view's) feature space, d = self.d columns, transform applied on the device
    def _centers(self, centers) -> np.ndarray:
        c = np.ascontiguousarray(centers, dtype=np.float64)
        if c.ndim != 2 or c.shape[0] < 1 or c.shape[1] != self.d:
            raise ValueError(f"centres have shape {c.shape}, data has {self.d} features")
        return c

    def kmeans_step(self, centers, sums: bool = True):
        """One Lloyd step over every shard of the world (agd_kmeans_step; collective: every rank gets the same bits):
        (sums, counts, cost) -- each centre's sum of its rows ((k, d), None unless `sums`) and their count, and the sum of every
        row's squared distance to its centre."""
        c = self._centers(centers)
        k = c.shape[0]
        s = np.empty((k, self.d), dtype=np.float64) if sums else None
        counts = np.empty(k, dtype=np.float64)
        cost = C.c_double()
        self._ensure_exchange()
        with self._filtered():
            N.check(N.lib().agd_kmeans_step(self.h, _ptr(c), k, _ptr(s), _ptr(counts), C.byref(cost)), self.h)
        return s, counts, cost.value

    def kmeans_costs(self, centers, keep: bool) -> float:
        """The k-means|| cost update (agd_kmeans_costs; collective): each row's cost becomes its squared distance to its
        closest of `centers`, or the smaller of that and its previous cost with `keep`; returns their sum over the world."""
        c = self._centers(centers)
        out = C.c_double()
        self._ensure_exchange()
        with self._filtered():
            N.check(N.lib().agd_kmeans_costs(self.h, _ptr(c), c.shape[0], 1 if keep else 0, C.byref(out)), self.h)
        return out.value

    def kmeans_sample(self, seed: int, factor: float, weighted: bool):
        """The rows kept by the k-means draw (agd_kmeans_sample; collective): u < factor * cost (weighted, the costs of the
        last kmeans_costs) or u < factor, with u the row's own draw under `seed`.  (rows (n, d), draws (n,)) in rank order."""
        L = N.lib()
        n = C.c_int64()
        self._ensure_exchange()
        with self._filtered():
            N.check(L.agd_kmeans_sample(self.h, int(seed) & (2 ** 64 - 1), float(factor), 1 if weighted else 0, 0, None, None,
                                        C.byref(n)), self.h)
            rows, draws = np.empty((n.value, self.d), dtype=np.float64), np.empty(n.value, dtype=np.float64)
            if n.value:
                N.check(L.agd_kmeans_sample(self.h, int(seed) & (2 ** 64 - 1), float(factor), 1 if weighted else 0, n.value,
                                            _ptr(rows), _ptr(draws), C.byref(n)), self.h)
        return rows, draws

    def kmeans_assign_rows(self, dev: int, row0: int, rows: int, centers):
        """Closest centre (-1 outside the view) and squared distance (NaN outside it) of physical rows [row0, row0 + rows) of
        local device `dev`'s shard (agd_kmeans_assign; not collective)."""
        c = self._centers(centers)
        cl = np.empty(max(int(rows), 0), dtype=np.int32)
        dist = np.empty(max(int(rows), 0), dtype=np.float64)
        with self._filtered():
            N.check(N.lib().agd_kmeans_assign(self.h, dev, _ptr(c), c.shape[0], int(row0), int(rows), _ptr(cl), _ptr(dist)),
                    self.h)
        return cl, dist

    def kmeans_assign(self, centers):
        """(cluster, distance) of this process's rows, across its local devices in load order (not collective); on a view, of
        the view's rows only, in the same order as margins."""
        cls, dists = [], []
        for i in range(len(self.ctx.devices)):
            cl, dist = self.kmeans_assign_rows(i, 0, self.local_rows(i), centers)
            keep = cl >= 0
            cls.append(cl[keep])
            dists.append(dist[keep])
        return np.concatenate(cls), np.concatenate(dists)

    # classification (agd_label_classes / agd_class_sums / agd_linear_*): labels compared by value, features in this dataset's
    # (or view's) space, d = self.d columns, transform applied on the device
    def _linear(self, W, offset):
        W = np.ascontiguousarray(W, dtype=np.float64)
        if W.ndim != 2 or W.shape[0] < 1 or W.shape[1] != self.d:
            raise ValueError(f"W has shape {W.shape}, data has {self.d} features")
        b = np.ascontiguousarray(offset, dtype=np.float64)
        if b.shape != (W.shape[0],):
            raise ValueError(f"offset has shape {b.shape}, W has {W.shape[0]} rows")
        return W, b

    @staticmethod
    def _classes(labels) -> np.ndarray:
        c = np.ascontiguousarray(labels, dtype=np.float64)
        if c.ndim != 1:
            raise ValueError(f"labels must be a vector, got shape {c.shape}")
        return c + 0.0   # -0.0 -> 0.0

    def label_classes(self):
        """The distinct labels of the rows over every shard of the world (agd_label_classes; collective: every rank gets the
        same values): (labels ascending, their counts (int64), rows whose label is NaN).  -0.0 is counted as 0.0."""
        L = N.lib()
        n, nan = C.c_int64(), C.c_int64()
        self._ensure_exchange()
        with self._filtered():
            N.check(L.agd_label_classes(self.h, 0, None, None, C.byref(n), C.byref(nan)), self.h)
            labels, counts = np.empty(n.value, dtype=np.float64), np.empty(n.value, dtype=np.int64)
            if n.value:
                N.check(L.agd_label_classes(self.h, n.value, _ptr(labels), _ptr(counts), C.byref(n), C.byref(nan)), self.h)
        return labels, counts, int(nan.value)

    def class_sums(self, labels):
        """Per class label (ascending, distinct, not NaN) over every shard of the world (agd_class_sums; collective):
        (sums (C, d) of the features of the rows with that label, their counts, entries of those rows that are not >= 0)."""
        c = self._classes(labels)
        sums = np.empty((c.shape[0], self.d), dtype=np.float64)
        counts = np.empty(c.shape[0], dtype=np.float64)
        neg = C.c_double()
        self._ensure_exchange()
        with self._filtered():
            N.check(N.lib().agd_class_sums(self.h, _ptr(c), c.shape[0], _ptr(sums), _ptr(counts), C.byref(neg)), self.h)
        return sums, counts, int(neg.value)

    def linear_argmax_rows(self, dev: int, row0: int, rows: int, W, offset) -> np.ndarray:
        """The lowest c maximising offset_c + x . W_c (-1 outside the view) of physical rows [row0, row0 + rows) of local
        device `dev`'s shard (agd_linear_argmax; not collective)."""
        W, b = self._linear(W, offset)
        cl = np.empty(max(int(rows), 0), dtype=np.int32)
        with self._filtered():
            N.check(N.lib().agd_linear_argmax(self.h, dev, _ptr(W), W.shape[0], _ptr(b), int(row0), int(rows), _ptr(cl)),
                    self.h)
        return cl

    def linear_argmax(self, W, offset) -> np.ndarray:
        """The argmax class of this process's rows, across its local devices in load order (not collective); on a view, of
        the view's rows only, in the same order as margins."""
        parts = []
        for i in range(len(self.ctx.devices)):
            cl = self.linear_argmax_rows(i, 0, self.local_rows(i), W, offset)
            parts.append(cl[cl >= 0])
        return np.concatenate(parts)

    def linear_confusion(self, W, offset, labels) -> np.ndarray:
        """(L, C) exact counts of the rows over every shard of the world (agd_linear_confusion; collective) by (index of
        their label in `labels`, argmax class); rows whose label is none of `labels` are not counted."""
        W, b = self._linear(W, offset)
        c = self._classes(labels)
        out = np.empty((c.shape[0], W.shape[0]), dtype=np.float64)
        self._ensure_exchange()
        with self._filtered():
            N.check(N.lib().agd_linear_confusion(self.h, _ptr(W), W.shape[0], _ptr(b), _ptr(c), c.shape[0], _ptr(out)),
                    self.h)
        return out

    def prox(self, updater: Updater, w, g, step: float, reg: float):
        """applyProjector (AGD.scala:214-222): (regVal, newWeights)."""
        w = np.ascontiguousarray(w, dtype=np.float64)
        g = np.ascontiguousarray(g, dtype=np.float64)
        out = np.empty_like(w)
        rv = C.c_double()
        N.check(N.lib().agd_prox(self.h, _upd_kind(updater), _ptr(w), _ptr(g), step, reg, w.shape[0], _ptr(out),
                                 C.byref(rv)), self.h)
        return rv.value, out

    def close(self):
        if self._base is not None:   # a view owns nothing; dropping it leaves the parent's shards alone
            return
        if self.h is not None:
            N.lib().agd_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MLUtils:
    """org.apache.spark.mllib.util.MLUtils [mllib-1.3.0]: the ingest side of the path."""

    @staticmethod
    def parseLibSVMFile(path: str, numFeatures: int = -1):
        """Host-only parse: (labels, rowptr, indices, values, d) with zero-based indices."""
        L = N.lib()
        obj = C.c_void_p()
        rc = L.agd_libsvm_read(path.encode(), numFeatures, C.byref(obj))
        try:
            if rc != 0:
                raise ValueError(L.agd_libsvm_error(obj).decode())
            n, d, nnz = L.agd_libsvm_rows(obj), L.agd_libsvm_dim(obj), L.agd_libsvm_nnz(obj)

            def arr(ptr, count, ctype, dtype):
                if count == 0:
                    return np.zeros(0, dtype=dtype)
                return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=(count,)).astype(dtype, copy=True)

            return (arr(L.agd_libsvm_labels(obj), n, C.c_double, np.float64),
                    arr(L.agd_libsvm_rowptr(obj), n + 1, C.c_int64, np.int64),
                    arr(L.agd_libsvm_indices(obj), nnz, C.c_int32, np.int32),
                    arr(L.agd_libsvm_values(obj), nnz, C.c_double, np.float64), int(d))
        finally:
            L.agd_libsvm_free(obj)

    @staticmethod
    def loadLibSVMFile(sc: "Context", path: str, numFeatures: int = -1, store: str = "f64") -> "DeviceDataset":
        """loadLibSVMFile(sc, path, numFeatures): rows land as CSR shards on the context's GPUs."""
        ds = DeviceDataset(sc)
        N.check(N.lib().agd_load_libsvm(ds.h, path.encode(), numFeatures, _STORE[store]), ds.h)
        ds.total_rows = sum(ds.local_rows(i) for i in range(len(sc.devices)))
        return ds

    @staticmethod
    def appendBias(x):
        """MLUtils.appendBias: a constant 1.0 as the last feature.  On a host matrix (or vector) a new array; on a DeviceDataset
        a view with d + 1 features that rewrites no row (the intercept is the last weight of a model trained on it)."""
        if isinstance(x, DeviceDataset):
            return x._transformed(bias=True)
        from .glm import append_bias
        x = np.asarray(x)
        return append_bias(x) if x.ndim == 2 else append_bias(x[None, :])[0]

    @staticmethod
    def kFold(data: "DeviceDataset", numFolds: int, seed: int = DEFAULT_SPLIT_SEED) -> list:
        """MLUtils.kFold(rdd, numFolds, seed): numFolds (training, validation) pairs of views; validation i keeps the rows
        whose draw lies in [i / k, (i + 1) / k), training i is its complement."""
        k = int(numFolds)
        if k < 2:
            raise ValueError(f"kFold needs numFolds >= 2, got {numFolds}")
        out = []
        for i in range(k):
            lo, hi = i / k, (i + 1) / k
            out.append((data._view((int(seed), lo, hi, True)), data._view((int(seed), lo, hi, False))))
        return out


def physical_model(w, intercept: float, scale=None, bias: bool = False):
    """(w, intercept) of a model on appendBias(s o x) as a model on the stored x: (s o v, intercept + b), where v are the
    feature weights and b the bias column's weight (the last of w when bias)."""
    w = np.asarray(w, dtype=np.float64)
    v, b = (w[:-1], float(w[-1])) if bias else (w, 0.0)
    if scale is not None:
        v = v * np.asarray(scale, dtype=np.float64)
    return np.ascontiguousarray(v), float(intercept) + b


def physical_projection(B, offset=None, scale=None, bias: bool = False, d: Optional[int] = None):
    """A projection x -> x B + offset of appendBias(s o x) as one of the stored x: (diag(s) B[:d_stored], offset + B[d_stored])
    with the bias row folded into the offset when bias (as physical_model folds a model).  B is (d, k) with d the view's
    width; a wrong shape, k < 1 or a non-finite entry (also one the fold makes) raises ValueError."""
    B = np.asarray(B, dtype=np.float64)
    if B.ndim != 2 or B.shape[1] < 1 or (d is not None and B.shape[0] != d):
        raise ValueError(f"B has shape {B.shape}; it must be (d, k) with d = {d} rows and k >= 1 columns")
    k = B.shape[1]
    c = np.zeros(k) if offset is None else np.asarray(offset, dtype=np.float64)
    if c.shape != (k,):
        raise ValueError(f"offset has shape {c.shape}; it must be ({k},)")
    if not (np.all(np.isfinite(B)) and np.all(np.isfinite(c))):
        raise ValueError("B and offset must be finite")
    P = B[:-1] if bias else B
    if bias:
        c = c + B[-1]
    if scale is not None:
        with np.errstate(over="ignore", invalid="ignore"):
            P = P * np.asarray(scale, dtype=np.float64)[:, None]
    if not (np.all(np.isfinite(P)) and np.all(np.isfinite(c))):
        raise ValueError("the projection of the stored features overflows (scale times B is not finite)")
    return np.ascontiguousarray(P), np.ascontiguousarray(c)


def _ratio(a: float, b: float) -> float:
    return a / b if b != 0 else float("nan")


@dataclass(frozen=True)
class Evaluation:
    """The sums agd_evaluate reduces over the world (AGD_EVAL_*), and the metrics derived from them on the host.
    Confusion counts cover rows labelled exactly 0 or 1 under the logistic / hinge losses; e = margin - label."""
    count: float
    loss_sum: float
    tp: float
    fp: float
    tn: float
    fn: float
    sum_err: float
    sum_err2: float
    sum_abs_err: float
    sum_y: float
    sum_y2: float

    @classmethod
    def from_sums(cls, sums) -> "Evaluation":
        return cls(*(float(v) for v in np.asarray(sums, dtype=np.float64)[:N.EVAL_N]))

    @property
    def mean_loss(self) -> float:
        """loss_sum / count: the loss applySmooth reports (AGD.scala:207), with the intercept inside the margin."""
        return _ratio(self.loss_sum, self.count)

    @property
    def accuracy(self) -> float:
        return _ratio(self.tp + self.tn, self.tp + self.fp + self.tn + self.fn)

    @property
    def precision(self) -> float:
        return _ratio(self.tp, self.tp + self.fp)

    @property
    def recall(self) -> float:
        return _ratio(self.tp, self.tp + self.fn)

    @property
    def mse(self) -> float:
        return _ratio(self.sum_err2, self.count)

    @property
    def rmse(self) -> float:
        return float(np.sqrt(self.mse))

    @property
    def mae(self) -> float:
        return _ratio(self.sum_abs_err, self.count)

    @property
    def r2(self) -> float:
        """1 - SSE / (sum y^2 - (sum y)^2 / n)."""
        return 1.0 - _ratio(self.sum_err2, self.sum_y2 - _ratio(self.sum_y ** 2, self.count))


@dataclass
class RunStats:
    iterations: int
    passes: int
    backtracks: int
    restarts: int
    converged: bool
    stopped_nan: bool
    nonterminating: bool
    final_L: float
    final_theta: float
    seconds_total: float
    k1_ms_total: float
    k1_launches: int
    gpu_launches: int
    allreduce_ms_total: float
    device_ms_total: float
    collective_calls: int
    collective_kind: int = 0
    fused_passes: int = 0      # evaluations that shared a sweep over X with another one (sweeps = passes - fused_passes)
    wasted_passes: int = 0


def _stats(st: N.Stats) -> RunStats:
    return RunStats(st.iterations, st.passes, st.backtracks, st.restarts, bool(st.converged), bool(st.stopped_nan),
                    bool(st.nonterminating), st.final_L, st.final_theta, st.seconds_total, st.k1_ms_total,
                    st.k1_launches, st.gpu_launches, st.allreduce_ms_total, st.device_ms_total, st.collective_calls, st.collective_kind,
                    st.fused_passes, st.wasted_passes)


# --------------------------------------------------------------------------- the optimizer
class AcceleratedGradientDescent:
    """class AcceleratedGradientDescent(gradient, updater) extends Optimizer (AGD.scala:41-144)."""

    def __init__(self, gradient: Gradient, updater: Updater):
        self.gradient = gradient
        self.updater = updater
        self.convergenceTol = 1e-4          # AGD.scala:44
        self.numIterations = 100            # :45
        self.regParam = 0.0                 # :46
        self.L0 = 1.0                       # :47
        self.Lexact = float("inf")          # :48
        self.beta = 0.5                     # :49
        self.alpha = 0.9                    # :50
        self.mayRestart = True              # :51
        self.memoize = False                # extension: AGD_FLAG_MEMOIZE_FX (bit-identical, fewer passes)
        self.fuse = True                    # pass fusion (AGD_FLAG_NO_FUSE clears it): same evaluations, fewer sweeps
        self.last_stats: Optional[RunStats] = None

    def setConvergenceTol(self, tol: float): self.convergenceTol = tol; return self       # :57
    def setNumIterations(self, iters: int): self.numIterations = iters; return self       # :65
    def setRegParam(self, regParam: float): self.regParam = regParam; return self         # :73
    def setL0(self, L0: float): self.L0 = L0; return self                                 # :78
    def setLexact(self, Lexact: float): self.Lexact = Lexact; return self                 # :83
    def setBeta(self, beta: float): self.beta = beta; return self                         # :88
    def setAlpha(self, alpha: float): self.alpha = alpha; return self                     # :93
    def setMayRestart(self, mayRestart: bool): self.mayRestart = mayRestart; return self  # :98
    def setGradient(self, gradient: Gradient): self.gradient = gradient; return self      # :106
    def setUpdater(self, updater: Updater): self.updater = updater; return self           # :117
    def setMemoize(self, on: bool): self.memoize = on; return self
    def setFuse(self, on: bool): self.fuse = on; return self

    def optimize(self, data: DeviceDataset, initialWeights) -> np.ndarray:                # :128-143
        w, _, st = run_with_stats(data, self.gradient, self.updater, self.convergenceTol, self.numIterations,
                                  self.regParam, initialWeights, self.L0, self.Lexact, self.beta, self.alpha,
                                  self.mayRestart, memoize=self.memoize, fuse=self.fuse)
        self.last_stats = st
        return w

    @staticmethod
    def run(data: DeviceDataset, gradient: Gradient, updater: Updater, convergenceTol: float, numIterations: int,
            regParam: float, initialWeights, L0: float, Lexact: float, beta: float, alpha: float,
            mayRestart: bool):
        """object AcceleratedGradientDescent.run (AGD.scala:177-189): returns (weights, lossHistory)."""
        w, hist, _ = run_with_stats(data, gradient, updater, convergenceTol, numIterations, regParam,
                                    initialWeights, L0, Lexact, beta, alpha, mayRestart)
        return w, hist


def run_with_stats(data: DeviceDataset, gradient, updater, convergenceTol, numIterations, regParam, initialWeights,
                   L0=1.0, Lexact=float("inf"), beta=0.5, alpha=0.9, mayRestart=True, memoize=False, fuse=True):
    if not isinstance(data, DeviceDataset):
        raise TypeError("data must be a DeviceDataset (Context.parallelize(...)); there is no CPU path")
    w0 = np.ascontiguousarray(initialWeights, dtype=np.float64)
    if w0.ndim != 1 or w0.shape[0] != data.d:
        raise ValueError(f"initialWeights has size {w0.shape}, data has {data.d} features")
    p = N.Params(convergenceTol, int(numIterations), regParam, L0, Lexact, beta, alpha, int(bool(mayRestart)),
                 _grad_kind(gradient), _upd_kind(updater), (N.FLAG_MEMOIZE_FX if memoize else 0) | (0 if fuse else N.FLAG_NO_FUSE))
    w = np.empty_like(w0)
    hist = np.empty(max(int(numIterations), 1), dtype=np.float64)
    nh, st = C.c_int32(), N.Stats()
    data._ensure_exchange()
    with data._filtered():
        N.check(N.lib().agd_run(data.h, C.byref(p), _ptr(w0), _ptr(w), _ptr(hist), C.byref(nh), C.byref(st)), data.h)
    return w, hist[:nh.value].copy(), _stats(st)


class GradientDescent:
    """GradientDescent.runMiniBatchSGD [mllib-1.3.0], the comparator of Suite.scala:78,118,225
    (miniBatchFraction < 1 samples rows with a counter-based Bernoulli mask keyed by 42 + i, see include/agd_b200.h)."""

    @staticmethod
    def runMiniBatchSGD(data: DeviceDataset, gradient: Gradient, updater: Updater, stepSize: float, numIterations: int,
                        regParam: float, miniBatchFraction: float, initialWeights):
        if not isinstance(data, DeviceDataset):
            raise TypeError("data must be a DeviceDataset (Context.parallelize(...)); there is no CPU path")
        w0 = np.ascontiguousarray(initialWeights, dtype=np.float64)
        if w0.ndim != 1 or w0.shape[0] != data.d:   # the native side reads and writes agd_dim(h) doubles
            raise ValueError(f"initialWeights has size {w0.shape}, data has {data.d} features")
        w = np.empty_like(w0)
        hist = np.empty(max(int(numIterations), 1), dtype=np.float64)
        nh, st = C.c_int32(), N.Stats()
        data._ensure_exchange()
        with data._filtered():
            N.check(N.lib().agd_gd_run_minibatch(data.h, _grad_kind(gradient), _upd_kind(updater), stepSize,
                                                 int(numIterations), regParam, float(miniBatchFraction), _ptr(w0), _ptr(w),
                                                 _ptr(hist), C.byref(nh), C.byref(st)), data.h)
        return w, hist[:nh.value].copy()
