"""ctypes view of the C-ABI in include/mb200.h.

Python is test and benchmark tooling here, not the product: the product is
``mrbayes_b200/lib/libmb200.so`` (CUDA, sm_90a) called from MrBayes' C code through the
seam in ``mrbayes_b200/seam/``.  The same structs drive the CPU oracle
(``oracle/liboracle.so``, ``orc_`` prefix) so that tests can feed identical inputs to both.

Nothing in this module computes likelihoods; if ``libmb200.so`` is missing it raises.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ENGINE_LIB = ROOT / "mrbayes_b200" / "lib" / "libmb200.so"
ORACLE_LIB = ROOT / "oracle" / "liboracle.so"

MAX_STATES = 64
MAX_CATEGORIES = 20
NONE = -1
CONFIG_THROUGHPUT = 1        # mb200_instance_config.flags: favour throughput over single-call latency
CONFIG_VARIABLE_STATES = 2   # STANDARD-data division: per-pattern state counts (the *_Std kernel family)
KERNEL_NUC4, KERNEL_TENSOR, KERNEL_GENERIC, KERNEL_STD, KERNEL_TIPROBS, KERNEL_SETUP = range(6)
KERNEL_NUC4_PARAMS, KERNEL_NUC4_PER_EVAL = 6, 7      # 4-state sub-counts (include/mb200.h)
EIGEN_INLINE = -2
FLAG_NUC4_PINVAR_QUIRK = 1
FLAG_TIP_SHORTCUTS = 2
FLAG_RANGE_GUARD = 4
EVAL_OK = 0
EVAL_UNDERFLOW = 1
SUCCESS = 0
ERROR_NO_DEVICE = -4


class InstanceConfig(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "tip_count", "partials_count", "state_count", "pattern_count", "category_count",
        "matrix_count", "scaler_count", "eigen_count", "weight_rows", "device",
        "max_evaluations", "flags")]


class Operation(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "dest", "child1", "matrix1", "child2", "matrix2", "child3", "matrix3",
        "scale_write", "scale_remove")]


class MatrixUpdate(C.Structure):
    _fields_ = [("matrix", C.c_int), ("eigen", C.c_int), ("length", C.c_double)]


class Evaluation(C.Structure):
    _fields_ = [
        ("matrix_update_count", C.c_int),
        ("matrix_updates", C.POINTER(MatrixUpdate)),
        ("operation_count", C.c_int),
        ("operations", C.POINTER(Operation)),
        ("site_scaler_dst", C.c_int),
        ("site_scaler_src", C.c_int),
        ("root_buffer", C.c_int),
        ("weights_row", C.c_int),
        ("flags", C.c_int),
        ("p_invar", C.c_double),
        ("has_p_invar", C.c_int),
        ("category_rates", C.c_double * MAX_CATEGORIES),
        ("category_weights", C.c_double * MAX_CATEGORIES),
        ("state_freqs", C.c_double * MAX_STATES),
        ("inline_eigen", C.POINTER(C.c_double)),
    ]


OP_DTYPE = np.dtype([(n, "<i4") for n, _ in Operation._fields_])
MAT_DTYPE = np.dtype([("matrix", "<i4"), ("eigen", "<i4"), ("length", "<f8")])
assert OP_DTYPE.itemsize == C.sizeof(Operation) == 36
assert MAT_DTYPE.itemsize == C.sizeof(MatrixUpdate) == 16


class AbiError(RuntimeError):
    def __init__(self, fn: str, code: int, msg: str = ""):
        super().__init__(f"{fn} failed with code {code} {msg}")
        self.code = code


def _ptr(a: np.ndarray, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


class Library:
    """One loaded shared library exporting the mb200 verb set under ``prefix``."""

    def __init__(self, path: os.PathLike, prefix: str):
        path = Path(path)
        if not path.exists():
            raise FileNotFoundError(
                f"{path} is missing: build it first (python -c 'import __graft_entry__ as g; g.build()')")
        self.path = path
        self.prefix = prefix
        self.lib = C.CDLL(str(path), mode=C.RTLD_GLOBAL)
        self._declare()

    def fn(self, name):
        return getattr(self.lib, self.prefix + name)

    def has(self, name) -> bool:
        return hasattr(self.lib, self.prefix + name)

    def _declare(self):
        I, D, P = C.c_int, C.c_double, C.POINTER
        sig = {
            "create_instance": [P(InstanceConfig), P(I)],
            "finalize_instance": [I],
            "set_tip_states": [I, I, P(C.c_uint64)],
            "set_pattern_weights": [I, I, P(C.c_float)],
            "set_pattern_states": [I, P(I), P(I), P(I), I, I, I],
            "set_cijk": [I, I, P(D)],
            "set_eigen_decomposition": [I, I, P(D), P(D), P(D)],
            "set_rate_matrices": [I, I, I, P(D), P(D)],
            "evaluate": [I, P(Evaluation), I, P(D), P(I)],
            "get_partials": [I, I, P(C.c_float)],
            "set_partials": [I, I, P(C.c_float)],
            "get_transition_matrix": [I, I, P(C.c_float)],
            "get_scalers": [I, I, P(C.c_float)],
            "set_transition_matrix": [I, I, P(C.c_float)],
            "set_scalers": [I, I, P(C.c_float)],
            # engine only
            "update_transition_matrices": [I, P(MatrixUpdate), I, P(D), P(D)],
            "update_partials": [I, P(Operation), I, I],
            "reset_scalers": [I, I],
            "copy_scalers": [I, I, I],
            "root_log_likelihood": [I, I, I, I, P(D), P(D), I, D, I, P(D), P(I)],
            "pack_evaluations": [I, P(Evaluation), I, P(I)],
            "replay": [I, I],
            "replay_results": [I, I, P(D), P(I)],
            "replay_begin": [I, I],
            "replay_end": [I, P(D), P(I)],
            "free_batch": [I, I],
            "synchronize": [I],
            "get_stream": [I, P(C.c_void_p)],
            "get_launch_count": [I, P(C.c_longlong)],
            "get_kernel_launches": [I, I, P(C.c_longlong)],
            "set_kernel_timing": [I, I],
            "get_kernel_time": [I, P(D), P(I)],
            "device_count": [],
            "abi_version": [],
            # oracle only
            "set_arith": [I, I],
        }
        for name, args in sig.items():
            if self.has(name):
                f = self.fn(name)
                f.argtypes = args
                f.restype = I
        if self.has("version_string"):
            self.fn("version_string").restype = C.c_char_p
            self.fn("error_string").restype = C.c_char_p
            self.fn("error_string").argtypes = [C.c_int]
        if self.has("cl_updates"):
            self.fn("cl_updates").restype = C.c_longlong
            self.fn("cl_updates").argtypes = [C.c_int]
        if self.has("compress_patterns"):
            self.fn("compress_patterns").restype = C.c_int
            self.fn("compress_patterns").argtypes = [P(C.c_uint64), I, I, P(I), P(I), P(I)]

    def check(self, name, rc):
        if rc != SUCCESS:
            msg = ""
            if self.has("error_string"):
                msg = "(" + self.fn("error_string")(rc).decode() + ")"
            raise AbiError(self.prefix + name, rc, msg)


_libs: dict = {}


def engine_library() -> Library:
    """libmb200.so -- the CUDA engine.  Fails loudly when it has not been built."""
    if "engine" not in _libs:
        _libs["engine"] = Library(ENGINE_LIB, "mb200_")
    return _libs["engine"]


def oracle_library() -> Library:
    """oracle/liboracle.so -- CPU checker; tests / smoke / bench cpu_baseline only."""
    if "oracle" not in _libs:
        _libs["oracle"] = Library(ORACLE_LIB, "orc_")
    return _libs["oracle"]


class EvalSpec:
    """Host description of one evaluation (one LaunchLogLikeForDivision call).

    Holds numpy arrays so the ctypes ``Evaluation`` built from it stays valid."""

    __slots__ = ("mats", "ops", "site_dst", "site_src", "root", "weights_row", "flags",
                 "p_invar", "has_p_invar", "rates", "cat_weights", "freqs", "chain", "division",
                 "lnl_ref", "aborted", "inline_eigen")

    def __init__(self, mats=None, ops=None, site_dst=NONE, site_src=NONE, root=NONE, weights_row=0,
                 flags=0, p_invar=0.0, has_p_invar=0, rates=(), cat_weights=(), freqs=(),
                 chain=0, division=0, lnl_ref=None, aborted=0, inline_eigen=None):
        self.mats = np.ascontiguousarray(mats if mats is not None else np.zeros(0, MAT_DTYPE), MAT_DTYPE)
        self.ops = np.ascontiguousarray(ops if ops is not None else np.zeros(0, OP_DTYPE), OP_DTYPE)
        self.site_dst, self.site_src, self.root, self.weights_row = site_dst, site_src, root, weights_row
        self.flags, self.p_invar, self.has_p_invar = flags, float(p_invar), int(has_p_invar)
        self.rates = np.asarray(rates, np.float64)
        self.cat_weights = np.asarray(cat_weights, np.float64)
        self.freqs = np.asarray(freqs, np.float64)
        self.chain, self.division, self.lnl_ref, self.aborted = chain, division, lnl_ref, aborted
        self.inline_eigen = None if inline_eigen is None else np.ascontiguousarray(inline_eigen, np.float64)

    def fill(self, ev: Evaluation):
        ev.matrix_update_count = len(self.mats)
        ev.matrix_updates = _ptr(self.mats, MatrixUpdate) if len(self.mats) else None
        ev.operation_count = len(self.ops)
        ev.operations = _ptr(self.ops, Operation) if len(self.ops) else None
        ev.site_scaler_dst, ev.site_scaler_src = self.site_dst, self.site_src
        ev.root_buffer, ev.weights_row, ev.flags = self.root, self.weights_row, self.flags
        ev.p_invar, ev.has_p_invar = self.p_invar, self.has_p_invar
        for k, v in enumerate(self.rates):
            ev.category_rates[k] = v
        for k, v in enumerate(self.cat_weights):
            ev.category_weights[k] = v
        for s, v in enumerate(self.freqs):
            ev.state_freqs[s] = v
        ev.inline_eigen = _ptr(self.inline_eigen, C.c_double) if self.inline_eigen is not None else None

    @property
    def node_updates(self) -> int:
        return len(self.ops)


def make_eval_array(specs):
    arr = (Evaluation * len(specs))()
    for ev, sp in zip(arr, specs):
        sp.fill(ev)
    return arr


class Instance:
    """A data division on one GPU (engine) or in host memory (oracle)."""

    def __init__(self, lib: Library, *, tip_count, partials_count, state_count, pattern_count,
                 category_count, matrix_count, scaler_count, eigen_count, weight_rows=1, device=0,
                 max_evaluations=1, flags=0):
        self.lib = lib
        self.cfg = InstanceConfig(tip_count, partials_count, state_count, pattern_count, category_count,
                                  matrix_count, scaler_count, eigen_count, weight_rows, device,
                                  max_evaluations, flags)
        self.cijk_parts = max(1, (flags >> 8) & 0xff)       # MB200_CONFIG_CIJK_PARTS
        h = C.c_int(-1)
        lib.check("create_instance", lib.fn("create_instance")(C.byref(self.cfg), C.byref(h)))
        self.handle = h.value
        self.S, self.K, self.C = state_count, category_count, pattern_count
        self.variable_states = bool(flags & CONFIG_VARIABLE_STATES)
        self.state_counts = None
        self.matrix_length = None
        self.batch_sizes = {}           # packed batch -> its evaluation count

    # -- lifetime --------------------------------------------------------------------
    def close(self):
        if self.handle >= 0:
            self.lib.fn("finalize_instance")(self.handle)
            self.handle = -1

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _call(self, name, *args):
        self.lib.check(name, self.lib.fn(name)(self.handle, *args))

    def _results(self, name, n, *args):
        """name(handle, *args, lnL, status) with room for n results -> (lnL, status)"""
        lnl = np.zeros(n, np.float64)
        st = np.zeros(n, np.int32)
        self._call(name, *args, _ptr(lnl, C.c_double), _ptr(st, C.c_int))
        return lnl, st

    # -- static data -------------------------------------------------------------------
    def set_tip_states(self, tip: int, masks):
        m = np.ascontiguousarray(masks, np.uint64)
        assert m.shape == (self.C,)
        self._call("set_tip_states", tip, _ptr(m, C.c_uint64))

    def set_pattern_weights(self, row: int, w):
        w = np.ascontiguousarray(w, np.float32)
        assert w.shape == (self.C,)
        self._call("set_pattern_weights", row, _ptr(w, C.c_float))

    def set_pattern_states(self, state_counts, matrix_offsets, freq_offsets, matrix_length, dummy_patterns, uncompressed_sites):
        """Variable-state divisions: m->nStates / tiIndex / bsIndex, tiProbLength, numDummyChars, numUncompressedChars."""
        ns = np.ascontiguousarray(state_counts, np.int32)
        ti = np.ascontiguousarray(matrix_offsets, np.int32)
        bs = np.ascontiguousarray(freq_offsets, np.int32)
        assert ns.shape == ti.shape == bs.shape == (self.C,)
        self._call("set_pattern_states", _ptr(ns, C.c_int), _ptr(ti, C.c_int), _ptr(bs, C.c_int),
                   int(matrix_length), int(dummy_patterns), int(uncompressed_sites))
        self.state_counts, self.matrix_length = ns.copy(), int(matrix_length)

    def set_cijk(self, eigen: int, block):
        b = np.ascontiguousarray(block, np.float64)
        assert b.size == self.cijk_parts * (2 * self.S + self.S ** 3)
        self._call("set_cijk", eigen, _ptr(b, C.c_double))

    def set_eigen_decomposition(self, eigen: int, V, Vinv, lam):
        V = np.ascontiguousarray(V, np.float64)
        Vi = np.ascontiguousarray(Vinv, np.float64)
        lam = np.ascontiguousarray(lam, np.float64)
        self._call("set_eigen_decomposition", eigen, _ptr(V, C.c_double), _ptr(Vi, C.c_double), _ptr(lam, C.c_double))

    def set_rate_matrices(self, eigen: int, Q, pi, like: int = NONE):
        """Device eigensolver: Q = [parts, S, S] reversible rate matrices, pi = their stationary frequencies;
        like = a slot holding the eigensystem of nearby matrices (warm start) or NONE."""
        q = np.ascontiguousarray(Q, np.float64)
        f = np.ascontiguousarray(pi, np.float64)
        assert q.size == self.cijk_parts * self.S * self.S and f.size == self.S
        self._call("set_rate_matrices", eigen, int(like), _ptr(q, C.c_double), _ptr(f, C.c_double))

    def set_arith(self, arith: int):
        self._call("set_arith", arith)

    # -- evaluation ---------------------------------------------------------------------
    def evaluate(self, specs):
        if isinstance(specs, EvalSpec):
            specs = [specs]
        return self._results("evaluate", len(specs), make_eval_array(specs), len(specs))

    def evaluate_begin(self, specs):
        """First half of evaluate(): validate, pack, launch; returns at once (one in flight per instance)."""
        if isinstance(specs, EvalSpec):
            specs = [specs]
        self._pending = make_eval_array(specs)          # keep the host structs alive until end()
        self._pending_n = len(specs)
        self._call("evaluate_begin", self._pending, self._pending_n)

    def evaluate_end(self):
        out = self._results("evaluate_end", self._pending_n)
        self._pending = None
        return out

    def pack(self, specs) -> int:
        arr = make_eval_array(specs)
        b = C.c_int(-1)
        self._call("pack_evaluations", arr, len(specs), C.byref(b))
        self.batch_sizes[b.value] = len(specs)
        return b.value

    def replay(self, batch: int):
        self._call("replay", batch)

    def replay_results(self, batch: int, n: int):
        return self._results("replay_results", n, batch)

    def replay_begin(self, batch: int):
        """First half of replaying a packed batch, on the resident kernel when the engine admits it there;
        replay_end() collects the results (one evaluation in flight per instance)."""
        self._call("replay_begin", batch)
        self._pending_n = self.batch_sizes[batch]

    def replay_end(self):
        return self._results("replay_end", self._pending_n)

    def free_batch(self, batch: int):
        self._call("free_batch", batch)

    def synchronize(self):
        self._call("synchronize")

    def stream(self) -> int:
        p = C.c_void_p()
        self._call("get_stream", C.byref(p))
        return p.value or 0

    def kernel_launches(self, kind: int) -> int:
        n = C.c_longlong(0)
        self._call("get_kernel_launches", kind, C.byref(n))
        return n.value

    def launch_count(self) -> int:
        n = C.c_longlong(0)
        self._call("get_launch_count", C.byref(n))
        return n.value

    def set_kernel_timing(self, on: bool):
        self._call("set_kernel_timing", 1 if on else 0)

    def kernel_time(self):
        """-> (summed ms, launches) of the fused pruning kernel since the last call."""
        ms = C.c_double(0.0)
        n = C.c_int(0)
        self._call("get_kernel_time", C.byref(ms), C.byref(n))
        return ms.value, n.value

    # -- node-granular verbs --------------------------------------------------------------
    def update_transition_matrices(self, mats, rates, freqs):
        """P(t) of the branches in mats; freqs are the stationary rows of branches past TIME_MAX.  None sends NULL,
        which only variable-state instances accept."""
        mats = np.ascontiguousarray(mats, MAT_DTYPE)
        rates = np.ascontiguousarray(rates, np.float64)
        f = None if freqs is None else np.ascontiguousarray(freqs, np.float64)
        self._call("update_transition_matrices", _ptr(mats, MatrixUpdate), len(mats), _ptr(rates, C.c_double),
                   None if f is None else _ptr(f, C.c_double))

    def update_partials(self, ops, site_scaler=NONE):
        ops = np.ascontiguousarray(ops, OP_DTYPE)
        self._call("update_partials", _ptr(ops, Operation), len(ops), site_scaler)

    def reset_scalers(self, scaler: int):
        self._call("reset_scalers", scaler)

    def copy_scalers(self, dst: int, src: int):
        self._call("copy_scalers", dst, src)

    def root_log_likelihood(self, root, site_scaler, weights_row, freqs, cat_weights, has_p_invar=0,
                            p_invar=0.0, flags=0):
        f = np.ascontiguousarray(freqs, np.float64)
        w = np.ascontiguousarray(cat_weights, np.float64)
        lnl = C.c_double(0.0)
        st = C.c_int(0)
        self._call("root_log_likelihood", root, site_scaler, weights_row, _ptr(f, C.c_double), _ptr(w, C.c_double),
                   has_p_invar, p_invar, flags, C.byref(lnl), C.byref(st))
        return lnl.value, st.value

    # -- read-back ------------------------------------------------------------------------
    def get_partials(self, buffer: int) -> np.ndarray:
        if self.variable_states:        # ragged reference layout [k][c][nStates[c]], returned flat per category
            out = np.zeros((self.K, int(self.state_counts.sum())), np.float32)
            self._call("get_partials", buffer, _ptr(out, C.c_float))
            return out
        out = np.zeros((self.K, self.C, self.S), np.float32)
        self._call("get_partials", buffer, _ptr(out, C.c_float))
        return out

    def set_transition_matrix(self, matrix: int, block):
        """A caller-supplied P(t): [K, S, S] floats, or for variable-state divisions a block of matrix_length"""
        b = np.ascontiguousarray(block, np.float32)
        assert b.size == (self.matrix_length if self.variable_states else self.K * self.S * self.S)
        self._call("set_transition_matrix", matrix, _ptr(b, C.c_float))

    def set_partials(self, buffer: int, a):
        """[K, C, S] floats, or for variable-state divisions the ragged layout get_partials returns"""
        a = np.ascontiguousarray(a, np.float32)
        if self.variable_states:
            assert a.shape == (self.K, int(self.state_counts.sum()))
        else:
            assert a.shape == (self.K, self.C, self.S)
        self._call("set_partials", buffer, _ptr(a, C.c_float))

    def set_scalers(self, scaler: int, v):
        """a node or site scaler buffer: [C] floats"""
        v = np.ascontiguousarray(v, np.float32)
        assert v.shape == (self.C,)
        self._call("set_scalers", scaler, _ptr(v, C.c_float))

    def get_transition_matrix(self, matrix: int) -> np.ndarray:
        if self.variable_states:
            out = np.zeros(self.matrix_length, np.float32)
            self._call("get_transition_matrix", matrix, _ptr(out, C.c_float))
            return out
        out = np.zeros((self.K, self.S, self.S), np.float32)
        self._call("get_transition_matrix", matrix, _ptr(out, C.c_float))
        return out

    def get_scalers(self, scaler: int) -> np.ndarray:
        out = np.zeros(self.C, np.float32)
        self._call("get_scalers", scaler, _ptr(out, C.c_float))
        return out
