"""ctypes binding of libtvm_b200.so (include/tvm_b200.h) — the Python-side mirror used by the
tests, bench.py and the multi-GPU driver.  PyTorch is used only for device memory, streams and
torch.distributed plumbing; all arithmetic happens in the CUDA library.

There is NO CPU fallback: if the library or a CUDA device is missing, creating a `Backend`
raises `TvmError`.
"""
import ctypes
import os
import subprocess
import sys
import numpy as np

_PKG = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))  # triton-vm_b200/
LIB_PATH = os.environ.get("TVM_B200_LIB") or os.path.join(_PKG, "lib", "libtvm_b200.so")  # override: A/B builds only
P = (1 << 64) - (1 << 32) + 1

_u64p = ctypes.POINTER(ctypes.c_uint64)
_vp = ctypes.c_void_p


class TvmError(RuntimeError):
    def __init__(self, code, msg=""):
        self.code = code
        super().__init__(f"libtvm_b200 error {code}: {msg}")


def build(force=False, verbose=False):
    """Compile libtvm_b200.so for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    args = ["make", "-C", _PKG, "-j8", "PYTHON=" + sys.executable, "lib/libtvm_b200.so"]   # the generators run on this interpreter
    if force:
        args.insert(1, "-B")
    r = subprocess.run(args, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building libtvm_b200.so failed:\n" + r.stdout[-4000:] + r.stderr[-4000:])
    if verbose:
        print(r.stdout[-2000:])
    return LIB_PATH


class Params(ctypes.Structure):
    _fields_ = [("security_level", ctypes.c_uint32), ("log2_ldt_expansion_factor", ctypes.c_uint32), ("ldt_choice", ctypes.c_uint32),
                ("soundness", ctypes.c_uint32)]


class Domains(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint64) for n in (
        "padded_height", "num_trace_randomizers", "randomized_trace_len", "trace_len", "quotient_len", "ldt_len",
        "ldt_offset", "num_collinearity_checks", "fri_num_rounds", "fri_last_round_max_degree",
        "num_quotient_randomizer_coefficients", "ldt", "num_first_round_queries", "stir_num_rounds")] + [
        ("stir_in_domain_queries", ctypes.c_uint64 * 16), ("stir_out_of_domain_queries", ctypes.c_uint64 * 16),
        ("stir_final_num_queries", ctypes.c_uint64), ("stir_final_degree", ctypes.c_uint64)]

    def as_dict(self):
        d = {}
        for n, t in self._fields_:
            v = getattr(self, n)
            d[n] = int(v) if t is ctypes.c_uint64 else [int(x) for x in v]
        k = d["stir_num_rounds"]
        d["stir_round_queries"] = list(zip(d.pop("stir_in_domain_queries")[:k], d.pop("stir_out_of_domain_queries")[:k]))
        return d


class FriInfo(ctypes.Structure):   # tvm_fri_info
    _fields_ = [(n, ctypes.c_uint64) for n in (
        "domain_len", "domain_offset", "expansion_factor", "max_degree", "num_collinearity_checks", "num_rounds", "last_round_max_degree")]


class ClaimStruct(ctypes.Structure):
    _fields_ = [("program_digest", ctypes.c_uint64 * 5), ("version", ctypes.c_uint32), ("input", _u64p),
                ("num_input", ctypes.c_size_t), ("output", _u64p), ("num_output", ctypes.c_size_t)]


class AetStruct(ctypes.Structure):   # tvm_aet (aet.rs:41-91)
    _fields_ = [("program", _u64p), ("program_len", ctypes.c_uint64),
                ("instruction_multiplicities", ctypes.POINTER(ctypes.c_uint32)),
                ("processor_trace", _u64p), ("processor_rows", ctypes.c_uint64),
                ("op_stack_underflow_trace", _u64p), ("op_stack_rows", ctypes.c_uint64),
                ("ram_trace", _u64p), ("ram_rows", ctypes.c_uint64),
                ("program_hash_trace", _u64p), ("program_hash_rows", ctypes.c_uint64),
                ("sponge_trace", _u64p), ("sponge_rows", ctypes.c_uint64),
                ("hash_trace", _u64p), ("hash_rows", ctypes.c_uint64),
                ("u32_entries", _u64p), ("u32_count", ctypes.c_uint64),
                ("cascade_table_lookup_multiplicities", _u64p), ("cascade_count", ctypes.c_uint64),
                ("lookup_table_lookup_multiplicities", _u64p)]


_AET_WIDTHS = dict(processor_trace=39, op_stack_underflow_trace=4, ram_trace=7, program_hash_trace=67, sponge_trace=67, hash_trace=67,
                   u32_entries=4, cascade_table_lookup_multiplicities=2)
_AET_COUNTS = dict(processor_trace="processor_rows", op_stack_underflow_trace="op_stack_rows", ram_trace="ram_rows",
                   program_hash_trace="program_hash_rows", sponge_trace="sponge_rows", hash_trace="hash_rows", u32_entries="u32_count",
                   cascade_table_lookup_multiplicities="cascade_count")


def aet_struct(arrays):
    """dict of numpy arrays named like the fields of tvm_aet -> (AetStruct, keep-alive list)"""
    keep = []
    s = AetStruct()
    prog = np.ascontiguousarray(arrays["program"], dtype=np.uint64)
    mult = np.ascontiguousarray(arrays["instruction_multiplicities"], dtype=np.uint32)
    assert prog.ndim == 1 and mult.shape == prog.shape
    keep += [prog, mult]
    s.program, s.program_len = prog.ctypes.data_as(_u64p), prog.size
    s.instruction_multiplicities = mult.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32))
    for name, width in _AET_WIDTHS.items():
        x = arrays[name]
        if hasattr(x, "data_ptr"):                      # contiguous torch tensor (pinned host or CUDA): [rows, width] 8-byte words
            assert x.is_contiguous() and x.element_size() == 8 and (x.numel() == 0 or x.shape[-1] == width)
            keep.append(x)
            setattr(s, name, ctypes.cast(x.data_ptr(), _u64p))
            setattr(s, _AET_COUNTS[name], x.numel() // width)
            continue
        a = np.ascontiguousarray(x, dtype=np.uint64).reshape(-1, width)
        keep.append(a)
        setattr(s, name, a.ctypes.data_as(_u64p))
        setattr(s, _AET_COUNTS[name], a.shape[0])
    lk = np.ascontiguousarray(arrays["lookup_table_lookup_multiplicities"], dtype=np.uint64)
    assert lk.shape == (256,)
    keep.append(lk)
    s.lookup_table_lookup_multiplicities = lk.ctypes.data_as(_u64p)
    return s, keep


class NondeterminismStruct(ctypes.Structure):   # tvm_nondeterminism (vm.rs:1467-1471)
    _fields_ = [("individual_tokens", _u64p), ("num_individual_tokens", ctypes.c_size_t), ("digests", _u64p),
                ("num_digests", ctypes.c_size_t), ("ram_addresses", _u64p), ("ram_values", _u64p), ("num_ram", ctypes.c_size_t)]


class ExecutionSummary(ctypes.Structure):   # tvm_execution_summary
    _fields_ = [("program_digest", ctypes.c_uint64 * 5), ("padded_height", ctypes.c_uint64), ("table_heights", ctypes.c_uint64 * 9),
                ("num_output", ctypes.c_uint64)]


TABLES = ("program", "processor", "op_stack", "ram", "jump_stack", "hash", "cascade", "lookup", "u32")   # table_heights order
TVM_ERR_VM = -10
CURRENT_VERSION = 6


AUX_CALLBACK = ctypes.CFUNCTYPE(ctypes.c_int, _vp, _u64p, ctypes.POINTER(_u64p), ctypes.POINTER(_u64p))
ALL_GATHER_CB = ctypes.CFUNCTYPE(ctypes.c_int, _vp, _vp, ctypes.c_size_t, _vp)
ALL_REDUCE_CB = ctypes.CFUNCTYPE(ctypes.c_int, _vp, _u64p, ctypes.c_size_t, _vp)


class CommStruct(ctypes.Structure):   # tvm_comm
    _fields_ = [("rank", ctypes.c_int), ("world", ctypes.c_int), ("user", _vp), ("all_gather", ALL_GATHER_CB),
                ("all_reduce_sum_u64", ALL_REDUCE_CB)]


LDT_AUTO, LDT_FRI, LDT_STIR = 0, 1, 2      # tvm_params.ldt_choice


class AirConstraintStruct(ctypes.Structure):   # tvm_air_constraint
    _fields_ = [(n, ctypes.c_uint32) for n in ("category", "index_in_category", "degree", "origin", "origin_index", "derived_column")] + \
        [("origin_name", ctypes.c_char_p)]


_U64x604 = ctypes.c_uint64 * 604

_lib = None
NUM_MAIN_COLUMNS, NUM_AUX_COLUMNS, NUM_CHALLENGES = 379, 91, 63      # include/tvm_b200.h

# name -> (restype, argtypes); every symbol declared in include/tvm_b200.h
_SIGNATURES = {
    "tvm_ctx_create": (ctypes.c_int, [ctypes.POINTER(_vp), ctypes.c_int]),
    "tvm_ctx_destroy": (None, [_vp]),
    "tvm_ctx_set_stream": (ctypes.c_int, [_vp, _vp]),
    "tvm_ctx_synchronize": (ctypes.c_int, [_vp]),
    "tvm_ctx_set_comm": (ctypes.c_int, [_vp, ctypes.POINTER(CommStruct)]),
    "tvm_ctx_set_low_memory": (ctypes.c_int, [_vp, ctypes.c_int]),
    "tvm_last_prove_low_memory": (ctypes.c_int, [_vp]),
    "tvm_strerror": (ctypes.c_char_p, [ctypes.c_int]),
    "tvm_last_error": (ctypes.c_char_p, [_vp]),
    "tvm_launch_count": (ctypes.c_uint64, [_vp]),
    "tvm_device_count": (ctypes.c_int, []),
    "tvm_to_mont_dev": (ctypes.c_int, [_vp, _vp, ctypes.c_size_t]),
    "tvm_from_mont_dev": (ctypes.c_int, [_vp, _vp, ctypes.c_size_t]),
    "tvm_ntt_bfe_dev": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_uint, ctypes.c_size_t, ctypes.c_int]),
    "tvm_ntt_bfe": (ctypes.c_int, [_vp, _u64p, ctypes.c_uint, ctypes.c_size_t, ctypes.c_int]),
    "tvm_lde_bfe_dev": (ctypes.c_int, [_vp, _vp, _vp, ctypes.c_uint, ctypes.c_uint, ctypes.c_uint, ctypes.c_uint64,
                                       ctypes.c_size_t, _vp, _vp, _vp]),
    "tvm_lde_bfe": (ctypes.c_int, [_vp, _u64p, _u64p, ctypes.c_uint, ctypes.c_uint, ctypes.c_uint, ctypes.c_uint64,
                                   ctypes.c_size_t, _u64p]),
    "tvm_tip5_hash_rows_dev": (ctypes.c_int, [_vp, _vp, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint, ctypes.c_uint, _vp]),
    "tvm_tip5_hash_rows": (ctypes.c_int, [_vp, _u64p, ctypes.c_size_t, ctypes.c_uint, _u64p]),
    "tvm_tip5_hash_varlen": (ctypes.c_int, [_u64p, ctypes.c_size_t, _u64p]),
    "tvm_merkle_build_dev": (ctypes.c_int, [_vp, _vp, ctypes.c_size_t]),
    "tvm_merkle_build": (ctypes.c_int, [_vp, _u64p, ctypes.c_size_t, _u64p, _u64p]),
    "tvm_derive_domains": (ctypes.c_int, [ctypes.POINTER(Params), ctypes.c_uint64, ctypes.POINTER(Domains)]),
    "tvm_prove": (ctypes.c_int, [_vp, ctypes.POINTER(Params), ctypes.POINTER(ClaimStruct), ctypes.c_uint64, _u64p, _u64p,
                                 AUX_CALLBACK, _vp, _u64p, _u64p, ctypes.POINTER(ctypes.c_size_t)]),
    "tvm_prove_tables": (ctypes.c_int, [_vp, ctypes.POINTER(Params), ctypes.POINTER(ClaimStruct), ctypes.c_uint64, _u64p, ctypes.c_int,
                                        _u64p, _u64p, _u64p, _u64p, _u64p, ctypes.POINTER(ctypes.c_size_t)]),
    "tvm_main_table_from_aet": (ctypes.c_int, [_vp, ctypes.POINTER(AetStruct), ctypes.c_uint64, _u64p, _u64p]),
    "tvm_prove_aet": (ctypes.c_int, [_vp, ctypes.POINTER(Params), ctypes.POINTER(ClaimStruct), ctypes.c_uint64, ctypes.POINTER(AetStruct),
                                     _u64p, _u64p, _u64p, _u64p, _u64p, ctypes.POINTER(ctypes.c_size_t)]),
    "tvm_bezout_coefficients": (ctypes.c_int, [_vp, _u64p, ctypes.c_uint64, _u64p, _u64p]),
    "tvm_prover_randomness": (ctypes.c_int, [_vp, ctypes.POINTER(Params), ctypes.c_uint64, ctypes.c_char_p, _u64p, _u64p, _u64p, _u64p]),
    "tvm_prove_aet_seeded": (ctypes.c_int, [_vp, ctypes.POINTER(Params), ctypes.POINTER(ClaimStruct), ctypes.c_uint64,
                                            ctypes.POINTER(AetStruct), ctypes.c_char_p, _u64p, ctypes.POINTER(ctypes.c_size_t)]),
    "tvm_prove_tables_seeded": (ctypes.c_int, [_vp, ctypes.POINTER(Params), ctypes.POINTER(ClaimStruct), ctypes.c_uint64, _u64p,
                                               ctypes.c_int, ctypes.c_char_p, _u64p, ctypes.POINTER(ctypes.c_size_t)]),
    "tvm_prove_transcript": (ctypes.c_int, [_vp, ctypes.POINTER(Params), ctypes.POINTER(ClaimStruct), ctypes.c_uint64, _u64p, _u64p,
                                            AUX_CALLBACK, _vp, _u64p, ctypes.c_void_p]),
    "tvm_stir_prove": (ctypes.c_int, [_vp, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, _u64p, _u64p,
                                      ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_size_t)]),
    "tvm_stir_verify": (ctypes.c_int, [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, _u64p, ctypes.c_size_t,
                                       ctypes.POINTER(ctypes.c_uint32), _u64p, ctypes.POINTER(ctypes.c_size_t), ctypes.c_char_p, ctypes.c_size_t]),
    "tvm_fri_derive": (ctypes.c_int, [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(FriInfo)]),
    "tvm_fri_prove": (ctypes.c_int, [_vp, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, _u64p, ctypes.c_size_t, _u64p,
                                     ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_size_t)]),
    "tvm_fri_verify": (ctypes.c_int, [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, _u64p, ctypes.c_size_t,
                                      ctypes.POINTER(ctypes.c_uint32), _u64p, ctypes.POINTER(ctypes.c_size_t), ctypes.c_char_p, ctypes.c_size_t]),
    "tvm_fill_derived_main_columns": (ctypes.c_int, [_vp, _u64p, ctypes.c_uint]),
    "tvm_aux_extend": (ctypes.c_int, [_vp, _u64p, ctypes.c_uint, _u64p, _u64p, _u64p]),
    "tvm_verify": (ctypes.c_int, [ctypes.POINTER(Params), ctypes.POINTER(ClaimStruct), _u64p, ctypes.c_size_t, ctypes.c_int,
                                  ctypes.c_char_p, ctypes.c_size_t]),
    "tvm_verify_batch": (ctypes.c_int, [ctypes.POINTER(Params), ctypes.POINTER(ClaimStruct), ctypes.POINTER(_u64p),
                                        ctypes.POINTER(ctypes.c_size_t), ctypes.c_size_t, ctypes.c_int, ctypes.c_uint,
                                        ctypes.POINTER(ctypes.c_int)]),
    "tvm_proof_padded_height": (ctypes.c_int, [_u64p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64)]),
    "tvm_last_prove_timings": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_float)]),
    "tvm_trace_execution": (ctypes.c_int, [_u64p, ctypes.c_size_t, _u64p, ctypes.c_size_t, ctypes.POINTER(NondeterminismStruct),
                                           ctypes.POINTER(_vp), ctypes.c_char_p, ctypes.c_size_t]),
    "tvm_execution_info": (ctypes.c_int, [_vp, ctypes.POINTER(ExecutionSummary), _u64p]),
    "tvm_execution_aet": (ctypes.c_int, [_vp, _vp, ctypes.POINTER(AetStruct)]),
    "tvm_prove_execution": (ctypes.c_int, [_vp, ctypes.POINTER(Params), _vp, ctypes.c_char_p, _u64p, ctypes.POINTER(ctypes.c_size_t)]),
    "tvm_execution_destroy": (None, [_vp]),
    "tvm_air_quotient_dev": (ctypes.c_int, [_vp, _vp, ctypes.c_size_t, _vp, ctypes.c_size_t, _u64p, _u64p, ctypes.c_uint,
                                            ctypes.c_uint, ctypes.c_uint64, _vp, ctypes.c_size_t]),
    "tvm_air_check": (ctypes.c_int, [_vp, _u64p, _u64p, ctypes.c_uint, _u64p, _u64p, _u64p, _u64p, _u64p]),
    "tvm_air_check_aet": (ctypes.c_int, [_vp, ctypes.POINTER(AetStruct), ctypes.POINTER(ClaimStruct), ctypes.c_uint64, _u64p, _u64p, _u64p,
                                         _u64p, _u64p]),
    "tvm_air_check_execution": (ctypes.c_int, [_vp, _vp, _u64p, _u64p, _u64p, _u64p, _u64p]),
    "tvm_air_constraint_info": (ctypes.c_int, [ctypes.c_uint, ctypes.POINTER(AirConstraintStruct)]),
}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise TvmError(-2, f"{LIB_PATH} not built (run __graft_entry__.build()); no CPU fallback exists")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            f = getattr(l, name)  # AttributeError if the library does not export a declared symbol
            f.restype = res
            f.argtypes = args
        _lib = l
    return _lib


def stir_verify(security_level, log2_expansion, log2_high_degree_bound, proof, conjectured=False):
    """Stir::verify for arbitrary StirParameters (host code, no GPU) -> (accepted, failure, first-round indices, partial first codeword [k,3])"""
    pr, prp = _np_u64(proof)
    cap = ctypes.c_size_t(8192)
    idx = (ctypes.c_uint32 * 8192)()
    vals = np.zeros((8192, 3), dtype=np.uint64)
    msg = ctypes.create_string_buffer(256)
    rc = lib().tvm_stir_verify(security_level, int(conjectured), log2_expansion, log2_high_degree_bound, prp, pr.size, idx,
                               vals.ctypes.data_as(_u64p), ctypes.byref(cap), msg, 256)
    if rc == 0:
        k = cap.value
        return True, "", [int(idx[i]) for i in range(k)], vals[:k].copy()
    if rc == -9:
        return False, msg.value.decode(), [], vals[:0]
    raise TvmError(rc, lib().tvm_strerror(rc).decode())


def fri_derive(security_level, log2_expansion, log2_high_degree_bound, conjectured=False):
    """FriParameters::try_into_fri + Fri::{max_degree, num_rounds, last_round_max_degree} (host code, no GPU) -> dict of
    tvm_fri_info's fields; raises TvmError (TVM_ERR_LDT_PARAMS = -6) for parameters the reference rejects"""
    out = FriInfo()
    rc = lib().tvm_fri_derive(security_level, int(conjectured), log2_expansion, log2_high_degree_bound, ctypes.byref(out))
    if rc:
        raise TvmError(rc, lib().tvm_strerror(rc).decode())
    return {n: int(getattr(out, n)) for n, _ in FriInfo._fields_}


def fri_verify(security_level, log2_expansion, log2_high_degree_bound, proof, conjectured=False):
    """Fri::verify for arbitrary FriParameters (host code, no GPU) -> (accepted, failure, first-round indices, partial first
    codeword [k,3]).  Parameter errors raise TvmError."""
    pr, prp = _np_u64(proof)
    cap = 1 << 16
    icap = ctypes.c_size_t(cap)
    idx = (ctypes.c_uint32 * cap)()
    vals = np.zeros((cap, 3), dtype=np.uint64)
    msg = ctypes.create_string_buffer(256)
    rc = lib().tvm_fri_verify(security_level, int(conjectured), log2_expansion, log2_high_degree_bound, prp, pr.size, idx,
                              vals.ctypes.data_as(_u64p), ctypes.byref(icap), msg, 256)
    if rc == 0:
        k = icap.value
        return True, "", [int(idx[i]) for i in range(k)], vals[:k].copy()
    if rc == -9:
        return False, msg.value.decode(), [], vals[:0]
    raise TvmError(rc, lib().tvm_strerror(rc).decode() + " | " + msg.value.decode())


def _proof_capacity(dom):
    """upper bound of the proof length in words for the derived parameters `dom`"""
    nfq = dom["num_first_round_queries"]
    est = 64 + nfq * (379 + 273 + 15 + 3 * 40 * (dom["fri_num_rounds"] + 4)) + \
        3 * (dom["ldt_len"] >> dom["fri_num_rounds"]) * 2 + 3 * 470 * 2 + 4096
    if dom["ldt"] == LDT_STIR:   # per round: stacked leaves (4 XFE + framing) and authentication paths of every query
        height = dom["ldt_len"].bit_length()
        est += sum(q * (16 + 5 * height) + 64 for q, _ in dom["stir_round_queries"]) + \
            dom["stir_final_num_queries"] * (16 + 5 * height) + 3 * (dom["stir_final_degree"] + 2) + 1024
    return est


def _u64_arg(x):
    """(keepalive, u64 pointer, shape) of a numpy array or a contiguous torch tensor (host or device)."""
    if hasattr(x, "data_ptr"):
        assert x.is_contiguous() and x.element_size() == 8
        return x, ctypes.cast(x.data_ptr(), _u64p), tuple(x.shape)
    a, ap = _np_u64(x)
    return a, ap, tuple(a.shape)


def _np_u64(a):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return a, a.ctypes.data_as(_u64p)


def hash_varlen(words):
    """Tip5::hash_varlen on the host (no GPU needed)."""
    w, wp = _np_u64(np.array(words, dtype=np.uint64))
    d = np.zeros(5, dtype=np.uint64)
    rc = lib().tvm_tip5_hash_varlen(wp, w.size, d.ctypes.data_as(_u64p))
    if rc:
        raise TvmError(rc, lib().tvm_strerror(rc).decode())
    return [int(v) for v in d]


def _rows(ptr, count, width, dtype=np.uint64):
    """copy of `count` rows of `width` words at a ctypes pointer (NULL allowed when count == 0)"""
    if not count:
        return np.zeros((0, width) if width else 0, dtype=dtype)
    n = count * (width or 1)
    a = np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint32 if dtype == np.uint32 else ctypes.c_uint64)), shape=(n,))
    return a.copy().reshape((count, width) if width else (count,))


class Execution:
    """VM::trace_execution's result (tvm_trace_execution): program digest, padded height, table heights, public output, and the
    AlgebraicExecutionTrace on demand.  Host memory; `close()` frees it (also on garbage collection)."""

    def __init__(self, handle, public_input):
        self._l, self._h = lib(), handle
        s = ExecutionSummary()
        _check_plain(self._l.tvm_execution_info(self._h, ctypes.byref(s), None))
        out = np.zeros(max(1, int(s.num_output)), dtype=np.uint64)
        _check_plain(self._l.tvm_execution_info(self._h, ctypes.byref(s), out.ctypes.data_as(_u64p)))
        self.program_digest = [int(v) for v in s.program_digest]
        self.padded_height = int(s.padded_height)
        self.table_heights = dict(zip(TABLES, (int(v) for v in s.table_heights)))
        self.input = [int(v) for v in public_input]
        self.output = [int(v) for v in out[:int(s.num_output)]]

    @property
    def claim(self):
        """(program digest, input, output): the claim the other bindings take (Claim::new(digest).with_input().with_output())"""
        return (self.program_digest, self.input, self.output)

    def aet(self, backend=None):
        """the AET as a dict with tvm_aet's (and oracle.tracegen.aet_arrays's) keys; the three hash traces are expanded on
        `backend`'s device, and are None without a backend"""
        a = AetStruct()
        if backend is not None:
            backend._chk(self._l.tvm_execution_aet(backend._h, self._h, ctypes.byref(a)))
        else:
            _check_plain(self._l.tvm_execution_aet(None, self._h, ctypes.byref(a)))
        d = dict(program=_rows(a.program, a.program_len, 0),
                 instruction_multiplicities=_rows(a.instruction_multiplicities, a.program_len, 0, np.uint32),
                 lookup_table_lookup_multiplicities=_rows(a.lookup_table_lookup_multiplicities, 256, 0))
        for name, width in _AET_WIDTHS.items():
            count = getattr(a, _AET_COUNTS[name])
            ptr = getattr(a, name)
            d[name] = _rows(ptr, count, width) if (ptr or not count) else None
        return d

    def close(self):
        if getattr(self, "_h", None):
            self._l.tvm_execution_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _check_plain(rc, msg=""):
    if rc:
        raise TvmError(rc, lib().tvm_strerror(rc).decode() + (" | " + msg if msg else ""))


def trace_execution(words, public_input=(), secret_input=(), digests=(), ram=None):
    """VM::trace_execution on the host (no GPU): program words (Program::to_bwords()), public input, NonDeterminism (secret
    input, digests [k][5], initial RAM {address: value}) -> Execution.  A program the VM rejects raises TvmError with code
    TVM_ERR_VM (-10) and the reference's error variant in the message."""
    w, wp = _np_u64(np.array(list(words), dtype=np.uint64))
    i, ip = _np_u64(np.array(list(public_input), dtype=np.uint64))
    sec, sp = _np_u64(np.array(list(secret_input), dtype=np.uint64))
    dg, dp = _np_u64(np.array([list(d) for d in digests], dtype=np.uint64).reshape(-1, 5))
    ram = dict(ram or {})
    ra, rap = _np_u64(np.array(list(ram.keys()), dtype=np.uint64))
    rv, rvp = _np_u64(np.array(list(ram.values()), dtype=np.uint64))
    nd = NondeterminismStruct(sp, sec.size, dp, dg.shape[0], rap, rvp, ra.size)
    h = _vp()
    msg = ctypes.create_string_buffer(512)
    rc = lib().tvm_trace_execution(wp, w.size, ip, i.size, ctypes.byref(nd), ctypes.byref(h), msg, 512)
    _check_plain(rc, msg.value.decode())
    return Execution(h, [int(v) for v in i])


AIR_CATEGORIES = ("init", "cons", "tran", "term")
NUM_CONSTRAINTS = 604
_AIR_INFO = None


def air_constraint_info():
    """tvm_air_constraint_info for all 604 constraints of the evaluator order (host code, no GPU) -> list of dicts: index,
    category ("init" | "cons" | "tran" | "term"), index_in_category, degree, origin (the table's name, "GrandCrossTableArg"
    or "DegreeLowering"), origin_id (0..8 the tables in TABLES order, 9, 10), origin_index (an original constraint's position
    in its table's list before degree lowering; a substitution constraint's derived column) and derived_column (None, or
    ("main", column) / ("aux", column) for a substitution constraint)"""
    global _AIR_INFO
    if _AIR_INFO is None:
        out = []
        for j in range(NUM_CONSTRAINTS):
            c = AirConstraintStruct()
            _check_plain(lib().tvm_air_constraint_info(j, ctypes.byref(c)))
            out.append(dict(index=j, category=AIR_CATEGORIES[c.category], index_in_category=int(c.index_in_category), degree=int(c.degree),
                            origin=c.origin_name.decode(), origin_id=int(c.origin), origin_index=int(c.origin_index),
                            derived_column=(None, ("main", int(c.origin_index)), ("aux", int(c.origin_index)))[c.derived_column]))
        _AIR_INFO = out
    return [dict(d) for d in _AIR_INFO]


def _air_check_result(counts, first, last, arrays):
    """the outputs of a tvm_air_check* call -> (counts, first_rows, last_rows) numpy arrays, or the list of violated constraints"""
    c, f, l = (np.ctypeslib.as_array(x).copy() for x in (counts, first, last))
    if arrays:
        return c, f, l
    info = air_constraint_info()
    return [dict(info[j], count=int(c[j]), first_row=int(f[j]), last_row=int(l[j])) for j in np.nonzero(c)[0]]


def derive_domains(security_level=160, log2_expansion=2, padded_height=1 << 10, ldt_choice=LDT_AUTO, conjectured=False):
    """Stark::{fri, stir, max_degree, ...} + ProverDomains::derive; pure host function."""
    p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
    d = Domains()
    rc = lib().tvm_derive_domains(ctypes.byref(p), padded_height, ctypes.byref(d))
    if rc:
        raise TvmError(rc, lib().tvm_strerror(rc).decode())
    return d.as_dict()


def verify(claim, proof, security_level=160, log2_expansion=2, ldt_choice=LDT_AUTO, conjectured=False, skip_air_check=False):
    """Stark::verify (tvm_verify; host code, no GPU needed).  claim = (program_digest[5], input, output[, version]);
    proof: the proof words.  Returns (accepted: bool, failure: str) — failure names the reference's error variant."""
    digest, inp, out = claim[0], claim[1], claim[2]
    version = claim[3] if len(claim) > 3 else 6
    ia, iap = _np_u64(np.array(list(inp), dtype=np.uint64))
    oa, oap = _np_u64(np.array(list(out), dtype=np.uint64))
    cs = ClaimStruct((ctypes.c_uint64 * 5)(*[int(v) for v in digest]), version, iap, ia.size, oap, oa.size)
    p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
    pw, pwp = _np_u64(np.array(proof, dtype=np.uint64))
    buf = ctypes.create_string_buffer(256)
    rc = lib().tvm_verify(ctypes.byref(p), ctypes.byref(cs), pwp, pw.size, int(skip_air_check), buf, 256)
    if rc not in (0, -9):
        raise TvmError(rc, lib().tvm_strerror(rc).decode())
    return rc == 0, buf.value.decode()


def verify_batch(claims, proofs, security_level=160, log2_expansion=2, ldt_choice=LDT_AUTO, conjectured=False,
                 skip_air_check=False, num_threads=0):
    """tvm_verify_batch: independent proofs on host threads -> list of bool (accepted)"""
    assert len(claims) == len(proofs)
    keep, cs = [], (ClaimStruct * len(claims))()
    for i, claim in enumerate(claims):
        digest, inp, out = claim[0], claim[1], claim[2]
        ia, iap = _np_u64(np.array(list(inp), dtype=np.uint64))
        oa, oap = _np_u64(np.array(list(out), dtype=np.uint64))
        keep += [ia, oa]
        cs[i] = ClaimStruct((ctypes.c_uint64 * 5)(*[int(v) for v in digest]), claim[3] if len(claim) > 3 else 6, iap, ia.size, oap, oa.size)
    arrs = [np.ascontiguousarray(np.array(p_, dtype=np.uint64)) for p_ in proofs]
    ptrs = (_u64p * len(arrs))(*[a.ctypes.data_as(_u64p) for a in arrs])
    lens = (ctypes.c_size_t * len(arrs))(*[a.size for a in arrs])
    res = (ctypes.c_int * len(arrs))()
    p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
    rc = lib().tvm_verify_batch(ctypes.byref(p), cs, ptrs, lens, len(arrs), int(skip_air_check), num_threads, res)
    if rc not in (0, -9):
        raise TvmError(rc, lib().tvm_strerror(rc).decode())
    return [r == 0 for r in res]


def proof_padded_height(proof):
    """Proof::padded_height; raises TvmError if the proof does not decode or holds no / several Log2PaddedHeight items"""
    pw, pwp = _np_u64(np.array(proof, dtype=np.uint64))
    out = ctypes.c_uint64(0)
    rc = lib().tvm_proof_padded_height(pwp, pw.size, ctypes.byref(out))
    if rc:
        raise TvmError(rc, lib().tvm_strerror(rc).decode())
    return int(out.value)


class Backend:
    """One context = one GPU = one driving thread (mirrors Prover::prove being single-caller)."""

    def __init__(self, device=0):
        self._l = lib()
        h = _vp()
        rc = self._l.tvm_ctx_create(ctypes.byref(h), device)
        if rc:
            raise TvmError(rc, self._l.tvm_strerror(rc).decode())
        self._h = h
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            self._l.tvm_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc):
        if rc:
            raise TvmError(rc, self._l.tvm_strerror(rc).decode() + " | " + self._l.tvm_last_error(self._h).decode())

    @property
    def launches(self):
        return int(self._l.tvm_launch_count(self._h))

    def set_stream(self, cuda_stream_ptr):
        self._chk(self._l.tvm_ctx_set_stream(self._h, _vp(cuda_stream_ptr)))

    def synchronize(self):
        self._chk(self._l.tvm_ctx_synchronize(self._h))

    # ---- host-buffer (canonical) entry points ------------------------------------------
    def ntt(self, x, inverse=False):
        """x: [ncols, n] or [n] canonical uint64 -> same shape"""
        a = np.array(x, dtype=np.uint64, copy=True)
        shape = a.shape
        a2 = np.ascontiguousarray(a.reshape(-1, shape[-1]))
        n = a2.shape[1]
        self._chk(self._l.tvm_ntt_bfe(self._h, a2.ctypes.data_as(_u64p), n.bit_length() - 1, a2.shape[0], int(inverse)))
        return a2.reshape(shape)

    def lde(self, trace, rand, log2_cosets, offset):
        """trace [ncols, n]; rand [ncols, h] or None -> [ncols, n << log2_cosets] natural order"""
        t, tp = _np_u64(trace)
        ncols, n = t.shape
        if rand is not None:
            r, rp = _np_u64(rand)
            h = r.shape[1]
        else:
            rp, h = None, 0
        out = np.empty((ncols, n << log2_cosets), dtype=np.uint64)
        self._chk(self._l.tvm_lde_bfe(self._h, tp, rp, h, n.bit_length() - 1, log2_cosets, offset, ncols,
                                      out.ctypes.data_as(_u64p)))
        return out

    def hash_rows(self, table_colmajor):
        """table [ncols, nrows] -> digests [nrows, 5]"""
        t, tp = _np_u64(table_colmajor)
        ncols, nrows = t.shape
        d = np.empty((nrows, 5), dtype=np.uint64)
        self._chk(self._l.tvm_tip5_hash_rows(self._h, tp, nrows, ncols, d.ctypes.data_as(_u64p)))
        return d

    def merkle(self, leaves, want_nodes=False):
        l, lp = _np_u64(leaves)
        n = l.shape[0]
        root = np.empty(5, dtype=np.uint64)
        nodes = np.empty((2 * n, 5), dtype=np.uint64) if want_nodes else None
        self._chk(self._l.tvm_merkle_build(self._h, lp, n, nodes.ctypes.data_as(_u64p) if want_nodes else None,
                                           root.ctypes.data_as(_u64p)))
        return (root, nodes) if want_nodes else root

    def fill_derived_main_columns(self, main_trace):
        """DegreeLoweringTable::fill_derived_main_columns IN PLACE: main_trace [379, n] (writable C-contiguous numpy uint64
        array or contiguous torch tensor, host or this GPU); columns 149.. are overwritten from columns 0..148."""
        if isinstance(main_trace, np.ndarray):
            assert main_trace.dtype == np.uint64 and main_trace.flags["C_CONTIGUOUS"] and main_trace.flags["WRITEABLE"]
        keep, mp, shape = _u64_arg(main_trace)
        assert len(shape) == 2 and shape[0] == NUM_MAIN_COLUMNS and shape[1] & (shape[1] - 1) == 0
        self._chk(self._l.tvm_fill_derived_main_columns(self._h, mp, shape[1].bit_length() - 1))
        del keep
        return main_trace

    def aux_extend(self, main_trace, challenges, randomizer_column=None, out=None):
        """MasterMainTable::extend on the device: main_trace [379, n] canonical (numpy, or a contiguous torch tensor on
        the host or on this GPU), challenges [63, 3], randomizer_column [n, 3] (column 90) or None -> aux trace [91, n, 3]
        canonical.  `out`: optional preallocated destination (numpy or torch, host or device); a numpy array otherwise."""
        keep, mp, shape = _u64_arg(main_trace)
        assert len(shape) == 2 and shape[0] == NUM_MAIN_COLUMNS and shape[1] & (shape[1] - 1) == 0
        n = shape[1]
        ch = np.ascontiguousarray(np.asarray(challenges, dtype=np.uint64).reshape(63, 3))
        rp, rkeep = None, None
        if randomizer_column is not None:
            rkeep, rp, rshape = _u64_arg(randomizer_column)
            assert tuple(rshape) == (n, 3)
        if out is None:
            out = np.empty((NUM_AUX_COLUMNS, n, 3), dtype=np.uint64)
        okeep, op, oshape = _u64_arg(out)
        assert tuple(oshape) == (NUM_AUX_COLUMNS, n, 3)
        self._chk(self._l.tvm_aux_extend(self._h, mp, n.bit_length() - 1, ch.ctypes.data_as(_u64p), rp, op))
        del keep, rkeep, okeep
        return out

    def prove(self, claim, main_trace, main_rand, aux_provider, quot_rand, security_level=160, log2_expansion=2,
              padded_height=None, ldt_choice=LDT_AUTO, conjectured=False):
        """Stark::prove; `ldt_choice` LDT_AUTO (default: the reference's heuristic, what Stark::default() does) / LDT_FRI / LDT_STIR.  claim = (program_digest[5], input, output[, version]);
        main_trace [379, n], main_rand [379, h] canonical uint64; aux_provider(challenges [63,3]) ->
        (aux_trace [91, n, 3], aux_rand [91, h, 3]); quot_rand [(h+1)*5, 3].  Returns the proof words.
        The traces may be numpy arrays (host) or contiguous torch int64 tensors (pinned host or CUDA:
        the C ABI takes either kind of pointer)."""
        mt, mtp, mt_shape = _u64_arg(main_trace)
        mr, mrp, mr_shape = _u64_arg(main_rand)
        qr, qrp = _np_u64(quot_rand)
        n = mt_shape[1]
        ph = padded_height or n
        dom = derive_domains(security_level, log2_expansion, ph, ldt_choice, conjectured)
        h = dom["num_trace_randomizers"]
        assert mt_shape == (379, dom["trace_len"]) and mr_shape == (379, h), (mt_shape, mr_shape, dom)
        assert qr.size == 3 * dom["num_quotient_randomizer_coefficients"]
        digest, inp, out = claim[0], claim[1], claim[2]
        version = claim[3] if len(claim) > 3 else 6
        ia, iap = _np_u64(np.array(list(inp), dtype=np.uint64))
        oa, oap = _np_u64(np.array(list(out), dtype=np.uint64))
        cs = ClaimStruct((ctypes.c_uint64 * 5)(*[int(v) for v in digest]), version, iap, ia.size, oap, oa.size)
        err = []

        keep = []

        def cb(_user, ch_p, trace_pp, rand_pp):
            try:
                ch = np.ctypeslib.as_array(ch_p, shape=(63, 3)).copy()
                t, r = aux_provider(ch)
                t, tp, ts = _u64_arg(t)
                r, rp, rs = _u64_arg(r)
                assert int(np.prod(ts)) == 91 * n * 3 and int(np.prod(rs)) == 91 * h * 3, (ts, rs)
                keep.extend([t, r])           # redirect to the caller's buffers (zero copy)
                trace_pp[0] = tp
                rand_pp[0] = rp
                return 0
            except Exception as e:  # noqa: BLE001 - must not propagate through the C frame
                err.append(e)
                return 1

        p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
        cap = ctypes.c_size_t(0)
        est = _proof_capacity(dom)
        buf = np.empty(est, dtype=np.uint64)
        cap.value = est
        rc = self._l.tvm_prove(self._h, ctypes.byref(p), ctypes.byref(cs), ph, mtp, mrp, AUX_CALLBACK(cb), None, qrp,
                               buf.ctypes.data_as(_u64p), ctypes.byref(cap))
        if err:
            raise err[0]
        self._chk(rc)
        return buf[:cap.value].copy()

    def prove_transcript(self, claim, main_trace, main_rand, aux_provider, quot_rand, transcript, security_level=160, log2_expansion=2,
                         padded_height=None, ldt_choice=LDT_AUTO, conjectured=False):
        """tvm_prove_transcript: Stark::prove with the HOST keeping the proof stream.  `transcript` is any object with
        alter_fiat_shamir_state_with(words), enqueue_raw(variant, payload_words), sample_scalars(n) -> n triples,
        sample_indices(upper_bound, n) -> n ints (e.g. a subclass of oracle.codec.ProofStream in the tests)."""
        mt, mtp, mt_shape = _u64_arg(main_trace)
        mr, mrp, mr_shape = _u64_arg(main_rand)
        qr, qrp = _np_u64(quot_rand)
        n = mt_shape[1]
        ph = padded_height or n
        dom = derive_domains(security_level, log2_expansion, ph, ldt_choice, conjectured)
        h = dom["num_trace_randomizers"]
        digest, inp, out = claim[0], claim[1], claim[2]
        version = claim[3] if len(claim) > 3 else 6
        ia, iap = _np_u64(np.array(list(inp), dtype=np.uint64))
        oa, oap = _np_u64(np.array(list(out), dtype=np.uint64))
        cs = ClaimStruct((ctypes.c_uint64 * 5)(*[int(v) for v in digest]), version, iap, ia.size, oap, oa.size)
        err, keep = [], []

        def cb(_user, ch_p, trace_pp, rand_pp):
            try:
                t, r = aux_provider(np.ctypeslib.as_array(ch_p, shape=(63, 3)).copy())
                t, tp, ts = _u64_arg(t)
                r, rp, rs = _u64_arg(r)
                assert int(np.prod(ts)) == 91 * n * 3 and int(np.prod(rs)) == 91 * h * 3, (ts, rs)
                keep.extend([t, r])
                trace_pp[0] = tp
                rand_pp[0] = rp
                return 0
            except Exception as e:  # noqa: BLE001
                err.append(e)
                return 1

        def guard(fn):
            def wrapped(*a):
                try:
                    fn(*a)
                    return 0
                except Exception as e:  # noqa: BLE001 - must not propagate through the C frame
                    err.append(e)
                    return 1
            return wrapped

        F_ABS = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, _u64p, ctypes.c_size_t)
        F_ENQ = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_uint, _u64p, ctypes.c_size_t)
        F_SCA = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, _u64p)
        F_IDX = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_uint, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint))

        def f_abs(_u, w, k): transcript.alter_fiat_shamir_state_with([int(w[i]) for i in range(k)])
        def f_enq(_u, variant, w, k): transcript.enqueue_raw(int(variant), [int(w[i]) for i in range(k)])
        def f_sca(_u, k, out_p):
            for i, x in enumerate(transcript.sample_scalars(k)):
                out_p[3 * i], out_p[3 * i + 1], out_p[3 * i + 2] = int(x[0]), int(x[1]), int(x[2])
        def f_idx(_u, ub, k, out_p):
            for i, v in enumerate(transcript.sample_indices(int(ub), k)):
                out_p[i] = int(v)

        class T(ctypes.Structure):
            _fields_ = [("user", ctypes.c_void_p), ("abs", F_ABS), ("enq", F_ENQ), ("sca", F_SCA), ("idx", F_IDX)]
        ts_ = T(None, F_ABS(guard(f_abs)), F_ENQ(guard(f_enq)), F_SCA(guard(f_sca)), F_IDX(guard(f_idx)))
        p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
        rc = self._l.tvm_prove_transcript(self._h, ctypes.byref(p), ctypes.byref(cs), ph, mtp, mrp, AUX_CALLBACK(cb), None, qrp,
                                          ctypes.cast(ctypes.byref(ts_), ctypes.c_void_p))
        if err:
            raise err[0]
        self._chk(rc)

    def prove_tables(self, claim, main_table, main_rand, aux_rand, randomizer_column, quot_rand, security_level=160, log2_expansion=2,
                     padded_height=None, ldt_choice=LDT_AUTO, conjectured=False, fill_derived_main_columns=True):
        """tvm_prove_tables: Stark::prove with the table stages on the device — the degree-lowering main columns (when
        fill_derived_main_columns) and MasterMainTable::extend run inside the prove on the resident main trace.
        main_table [379, n] (columns 149.. ignored when they are filled on the device), main_rand [379, h], aux_rand [91, h, 3],
        randomizer_column [n, 3] or None, quot_rand [(h+1)*5, 3]; numpy or contiguous torch tensors (host or CUDA)."""
        mt, mtp, mt_shape = _u64_arg(main_table)
        mr, mrp, mr_shape = _u64_arg(main_rand)
        ar, arp, ar_shape = _u64_arg(aux_rand)
        qr, qrp = _np_u64(quot_rand)
        n = mt_shape[1]
        ph = padded_height or n
        dom = derive_domains(security_level, log2_expansion, ph, ldt_choice, conjectured)
        h = dom["num_trace_randomizers"]
        assert mt_shape == (379, dom["trace_len"]) and mr_shape == (379, h) and int(np.prod(ar_shape)) == 91 * h * 3, (mt_shape, mr_shape, ar_shape)
        assert qr.size == 3 * dom["num_quotient_randomizer_coefficients"]
        rcp = None
        if randomizer_column is not None:
            rc_, rcp, rc_shape = _u64_arg(randomizer_column)
            assert int(np.prod(rc_shape)) == 3 * n
        digest, inp, out = claim[0], claim[1], claim[2]
        version = claim[3] if len(claim) > 3 else 6
        ia, iap = _np_u64(np.array(list(inp), dtype=np.uint64))
        oa, oap = _np_u64(np.array(list(out), dtype=np.uint64))
        cs = ClaimStruct((ctypes.c_uint64 * 5)(*[int(v) for v in digest]), version, iap, ia.size, oap, oa.size)
        p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
        est = _proof_capacity(dom)
        buf = np.empty(est, dtype=np.uint64)
        cap = ctypes.c_size_t(est)
        rc = self._l.tvm_prove_tables(self._h, ctypes.byref(p), ctypes.byref(cs), ph, mtp, int(bool(fill_derived_main_columns)), mrp, arp,
                                      rcp, qrp, buf.ctypes.data_as(_u64p), ctypes.byref(cap))
        self._chk(rc)
        return buf[:cap.value].copy()

    def main_table_from_aet(self, aet, num_rows):
        """tvm_main_table_from_aet: MasterMainTable::new + pad + degree-lowering columns on the device.
        aet: dict of arrays named like tvm_aet's fields -> ([379, num_rows] canonical, the nine table lengths)"""
        s, keep = aet_struct(aet)
        out = np.empty((NUM_MAIN_COLUMNS, num_rows), dtype=np.uint64)
        lengths = np.zeros(9, dtype=np.uint64)
        rc = self._l.tvm_main_table_from_aet(self._h, ctypes.byref(s), num_rows, out.ctypes.data_as(_u64p), lengths.ctypes.data_as(_u64p))
        del keep
        self._chk(rc)
        return out, [int(v) for v in lengths]

    def bezout_coefficients(self, roots):
        """tvm_bezout_coefficients (ram.rs:162-214): distinct canonical roots -> (a, b) coefficient arrays"""
        r, rp = _np_u64(np.asarray(roots, dtype=np.uint64))
        a, b = np.zeros(r.size, dtype=np.uint64), np.zeros(r.size, dtype=np.uint64)
        self._chk(self._l.tvm_bezout_coefficients(self._h, rp, r.size, a.ctypes.data_as(_u64p), b.ctypes.data_as(_u64p)))
        return a, b

    def prove_aet(self, claim, aet, main_rand, aux_rand, randomizer_column, quot_rand, security_level=160, log2_expansion=2,
                  padded_height=None, ldt_choice=LDT_AUTO, conjectured=False):
        """tvm_prove_aet: Stark::prove from the AlgebraicExecutionTrace — table fill, padding, degree lowering, extension and
        the proof on the device.  aet: dict of arrays named like tvm_aet's fields; the rest as prove_tables."""
        s, keep = aet_struct(aet)
        mr, mrp, mr_shape = _u64_arg(main_rand)
        ar, arp, ar_shape = _u64_arg(aux_rand)
        qr, qrp = _np_u64(quot_rand)
        ph = int(padded_height)
        dom = derive_domains(security_level, log2_expansion, ph, ldt_choice, conjectured)
        h, n = dom["num_trace_randomizers"], dom["trace_len"]
        assert mr_shape == (379, h) and int(np.prod(ar_shape)) == 91 * h * 3, (mr_shape, ar_shape)
        assert qr.size == 3 * dom["num_quotient_randomizer_coefficients"]
        rcp = None
        if randomizer_column is not None:
            rc_, rcp, rc_shape = _u64_arg(randomizer_column)
            assert int(np.prod(rc_shape)) == 3 * n
        digest, inp, out = claim[0], claim[1], claim[2]
        version = claim[3] if len(claim) > 3 else 6
        ia, iap = _np_u64(np.array(list(inp), dtype=np.uint64))
        oa, oap = _np_u64(np.array(list(out), dtype=np.uint64))
        cs = ClaimStruct((ctypes.c_uint64 * 5)(*[int(v) for v in digest]), version, iap, ia.size, oap, oa.size)
        p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
        est = _proof_capacity(dom)
        buf = np.empty(est, dtype=np.uint64)
        cap = ctypes.c_size_t(est)
        rc = self._l.tvm_prove_aet(self._h, ctypes.byref(p), ctypes.byref(cs), ph, ctypes.byref(s), mrp, arp, rcp, qrp,
                                   buf.ctypes.data_as(_u64p), ctypes.byref(cap))
        del keep
        self._chk(rc)
        return buf[:cap.value].copy()

    @staticmethod
    def _seed(seed):
        """32 seed bytes (None passes NULL, which the library rejects)"""
        if seed is None:
            return None
        seed = bytes(seed)
        assert len(seed) == 32, "the prover's randomness seed is 32 bytes"
        return seed

    @staticmethod
    def _claim(claim):
        digest, inp, out = claim[0], claim[1], claim[2]
        version = claim[3] if len(claim) > 3 else 6
        ia, iap = _np_u64(np.array(list(inp), dtype=np.uint64))
        oa, oap = _np_u64(np.array(list(out), dtype=np.uint64))
        return ClaimStruct((ctypes.c_uint64 * 5)(*[int(v) for v in digest]), version, iap, ia.size, oap, oa.size), (ia, oa)

    def prover_randomness(self, seed, padded_height, security_level=160, log2_expansion=2, ldt_choice=LDT_AUTO, conjectured=False,
                          out=None):
        """tvm_prover_randomness: the prover's randomness drawn on the device from its 32-byte seed, as Prover::prove draws it
        -> (main_rand [379, h], aux_rand [91, h, 3], randomizer_column [n, 3], quot_rand [(h+1)*5, 3]), canonical.
        `out`: optional 4-tuple of destination arrays (numpy or contiguous torch tensors, host or CUDA; None skips one);
        by default four new numpy arrays."""
        dom = derive_domains(security_level, log2_expansion, padded_height, ldt_choice, conjectured)
        h, n, nq = dom["num_trace_randomizers"], dom["trace_len"], dom["num_quotient_randomizer_coefficients"]
        shapes = [(NUM_MAIN_COLUMNS, h), (NUM_AUX_COLUMNS, h, 3), (n, 3), (nq, 3)]
        if out is None:
            out = tuple(np.empty(s, dtype=np.uint64) for s in shapes)
        ptrs = []
        for o, s in zip(out, shapes):
            if o is None:
                ptrs.append(None)
                continue
            _, op, shape = _u64_arg(o)
            assert int(np.prod(shape)) == int(np.prod(s)), (shape, s)
            if isinstance(o, np.ndarray):
                assert o.flags.c_contiguous and o.dtype == np.uint64
            ptrs.append(op)
        p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
        self._chk(self._l.tvm_prover_randomness(self._h, ctypes.byref(p), padded_height, self._seed(seed), *ptrs))
        return out

    def prove_aet_seeded(self, claim, aet, seed, padded_height, security_level=160, log2_expansion=2, ldt_choice=LDT_AUTO,
                         conjectured=False):
        """tvm_prove_aet_seeded: Stark::prove from the AlgebraicExecutionTrace and the prover's 32-byte randomness seed alone —
        the proof Prover::prove gives with that seed.  The seed must come from a CSPRNG the verifier cannot predict."""
        s, keep = aet_struct(aet)
        ph = int(padded_height)
        dom = derive_domains(security_level, log2_expansion, ph, ldt_choice, conjectured)
        cs, keep_claim = self._claim(claim)
        p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
        est = _proof_capacity(dom)
        buf = np.empty(est, dtype=np.uint64)
        cap = ctypes.c_size_t(est)
        rc = self._l.tvm_prove_aet_seeded(self._h, ctypes.byref(p), ctypes.byref(cs), ph, ctypes.byref(s), self._seed(seed),
                                          buf.ctypes.data_as(_u64p), ctypes.byref(cap))
        del keep, keep_claim
        self._chk(rc)
        return buf[:cap.value].copy()

    def prove_execution(self, ex, seed, security_level=160, log2_expansion=2, ldt_choice=LDT_AUTO, conjectured=False):
        """tvm_prove_execution: Stark::prove of an Execution's claim from its AET (hash traces expanded on the device) and the
        prover's 32-byte randomness seed -> proof words.  The seed must come from a CSPRNG the verifier cannot predict."""
        dom = derive_domains(security_level, log2_expansion, ex.padded_height, ldt_choice, conjectured)
        p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
        est = _proof_capacity(dom)
        for _ in range(2):
            buf = np.empty(est, dtype=np.uint64)
            cap = ctypes.c_size_t(est)
            rc = self._l.tvm_prove_execution(self._h, ctypes.byref(p), ex._h, self._seed(seed), buf.ctypes.data_as(_u64p), ctypes.byref(cap))
            if rc == -1 and cap.value > est:    # the proof is longer than the estimate: prove again into a buffer that fits
                est = cap.value
                continue
            break
        self._chk(rc)
        return buf[:cap.value].copy()

    def prove_program(self, words, public_input=(), secret_input=(), digests=(), ram=None, seed=None, **params):
        """triton_vm::prove_program (lib.rs:228-267): trace the program on the host, prove on this GPU -> (claim, proof)"""
        ex = trace_execution(words, public_input, secret_input, digests, ram)
        try:
            return ex.claim, self.prove_execution(ex, seed, **params)
        finally:
            ex.close()

    # ---- AIR constraint check (tvm_air_check*) -------------------------------------------
    def air_check(self, main, aux, challenges, arrays=False):
        """tvm_air_check: every AIR constraint on the rows where it must vanish.  main [379, n], aux [91, n, 3] canonical (numpy,
        or contiguous torch tensors on the host or this GPU), challenges [63, 3] canonical -> the violated constraints (dicts of
        air_constraint_info() plus count, first_row, last_row), or with arrays=True (counts, first_rows, last_rows) [604] each"""
        km, mp, mshape = _u64_arg(main)
        ka, ap, ashape = _u64_arg(aux)
        assert len(mshape) == 2 and mshape[0] == NUM_MAIN_COLUMNS, mshape
        n = mshape[1]
        assert int(np.prod(ashape)) == NUM_AUX_COLUMNS * n * 3, ashape
        ch, chp = _np_u64(np.asarray(challenges, dtype=np.uint64).reshape(NUM_CHALLENGES, 3))
        out = [_U64x604() for _ in range(3)]
        nv = ctypes.c_uint64()
        self._chk(self._l.tvm_air_check(self._h, mp, ap, max(n.bit_length() - 1, 0), chp, *out, ctypes.byref(nv)))
        del km, ka
        return _air_check_result(*out, arrays)

    def air_check_aet(self, aet, claim, num_rows, sampled, arrays=False):
        """tvm_air_check_aet: the witness tvm_prove_aet builds from `aet` (fill, padding to num_rows, degree-lowering columns,
        Challenges::new from `claim` on the 59 sampled challenges [59, 3], extension) checked on the device; result as air_check"""
        s, keep = aet_struct(aet)
        cs, keep_claim = self._claim(claim)
        sp_, spp = _np_u64(np.asarray(sampled, dtype=np.uint64).reshape(59, 3))
        out = [_U64x604() for _ in range(3)]
        nv = ctypes.c_uint64()
        rc = self._l.tvm_air_check_aet(self._h, ctypes.byref(s), ctypes.byref(cs), int(num_rows), spp, *out, ctypes.byref(nv))
        del keep, keep_claim
        self._chk(rc)
        return _air_check_result(*out, arrays)

    def air_check_execution(self, ex, sampled, arrays=False):
        """tvm_air_check_execution: an Execution's witness at its padded height, checked on the device; result as air_check"""
        sp_, spp = _np_u64(np.asarray(sampled, dtype=np.uint64).reshape(59, 3))
        out = [_U64x604() for _ in range(3)]
        nv = ctypes.c_uint64()
        self._chk(self._l.tvm_air_check_execution(self._h, ex._h, spp, *out, ctypes.byref(nv)))
        return _air_check_result(*out, arrays)

    def check_program(self, words, public_input=(), secret_input=(), digests=(), ram=None, sampled=None, arrays=False):
        """trace the program on the host and check its witness against every AIR constraint on this GPU -> as air_check.
        `sampled`: the 59 sampled challenges [59, 3]; by default drawn with numpy from a fixed seed (a valid witness satisfies
        the AIR for every challenge value; the library draws no entropy)."""
        if sampled is None:
            sampled = np.random.default_rng(0x7A1C).integers(0, P, size=(59, 3), dtype=np.uint64)
        ex = trace_execution(words, public_input, secret_input, digests, ram)
        try:
            return self.air_check_execution(ex, sampled, arrays)
        finally:
            ex.close()

    def prove_tables_seeded(self, claim, main_table, seed, security_level=160, log2_expansion=2, padded_height=None, ldt_choice=LDT_AUTO,
                            conjectured=False, fill_derived_main_columns=True):
        """tvm_prove_tables_seeded: as prove_tables, with the randomness drawn on the device from the prover's 32-byte seed."""
        mt, mtp, mt_shape = _u64_arg(main_table)
        ph = padded_height or mt_shape[1]
        dom = derive_domains(security_level, log2_expansion, ph, ldt_choice, conjectured)
        assert mt_shape == (379, dom["trace_len"]), mt_shape
        cs, keep_claim = self._claim(claim)
        p = Params(security_level, log2_expansion, ldt_choice, int(conjectured))
        est = _proof_capacity(dom)
        buf = np.empty(est, dtype=np.uint64)
        cap = ctypes.c_size_t(est)
        rc = self._l.tvm_prove_tables_seeded(self._h, ctypes.byref(p), ctypes.byref(cs), ph, mtp, int(bool(fill_derived_main_columns)),
                                             self._seed(seed), buf.ctypes.data_as(_u64p), ctypes.byref(cap))
        del keep_claim
        self._chk(rc)
        return buf[:cap.value].copy()

    def stir_prove(self, security_level, log2_expansion, log2_high_degree_bound, codeword, conjectured=False):
        """Stir::prove on the device for arbitrary StirParameters: codeword [2^(hdb+exp), 3] canonical -> (proof words, revealed indices)"""
        cw, cwp, shape = _u64_arg(codeword)
        n = 1 << (log2_high_degree_bound + log2_expansion)
        assert int(np.prod(shape)) == 3 * n
        cap = ctypes.c_size_t(0)
        icap = ctypes.c_size_t(8192)
        idx = (ctypes.c_uint32 * 8192)()
        est = 1 << 22
        buf = np.empty(est, dtype=np.uint64)
        cap.value = est
        self._chk(self._l.tvm_stir_prove(self._h, security_level, int(conjectured), log2_expansion, log2_high_degree_bound, cwp,
                                         buf.ctypes.data_as(_u64p), ctypes.byref(cap), idx, ctypes.byref(icap)))
        return buf[:cap.value].copy(), [int(idx[i]) for i in range(icap.value)]

    def fri_prove(self, security_level, log2_expansion, log2_high_degree_bound, codeword, conjectured=False):
        """Fri::prove on the device for arbitrary FriParameters: codeword [2^(hdb+exp), 3] canonical (numpy, or a contiguous torch
        tensor on the host or the device) -> (proof words, first-round indices)"""
        cw, cwp, shape = _u64_arg(codeword)
        n = int(np.prod(shape)) // 3
        try:
            fd = fri_derive(security_level, log2_expansion, log2_high_degree_bound, conjectured)
        except TvmError:
            fd = dict(num_collinearity_checks=0, num_rounds=0, domain_len=0)   # tvm_fri_prove names the parameter error
        checks, rounds = fd["num_collinearity_checks"], fd["num_rounds"]
        # roots, last codeword and polynomial, one response per round: leaves plus at most checks * height digests
        est = 64 + 8 * (rounds + 1) + 6 * (fd["domain_len"] >> rounds) + (rounds + 1) * (8 + checks * (3 + 5 * fd["domain_len"].bit_length()))
        buf = np.empty(est, dtype=np.uint64)
        cap = ctypes.c_size_t(est)
        icap = ctypes.c_size_t(max(1, checks))
        idx = (ctypes.c_uint32 * max(1, checks))()
        self._chk(self._l.tvm_fri_prove(self._h, security_level, int(conjectured), log2_expansion, log2_high_degree_bound, cwp, n,
                                        buf.ctypes.data_as(_u64p), ctypes.byref(cap), idx, ctypes.byref(icap)))
        return buf[:cap.value].copy(), [int(idx[i]) for i in range(icap.value)]

    def set_low_memory(self, mode):
        """0 = automatic, 1 = always just-in-time LDE (tables never stored), 2 = always cache."""
        self._chk(self._l.tvm_ctx_set_low_memory(self._h, int(mode)))

    @property
    def last_prove_low_memory(self):
        return bool(self._l.tvm_last_prove_low_memory(self._h))

    def set_comm(self, comm):
        """Attach a communication layer (tvm_b200.dist.TorchDistComm) so that prove() shards one proof over
        the ranks of its process group; None detaches."""
        if comm is None:
            self._chk(self._l.tvm_ctx_set_comm(self._h, None))
            self._comm = None
            return
        cs = comm.as_struct()
        self._chk(self._l.tvm_ctx_set_comm(self._h, ctypes.byref(cs)))
        self._comm = (comm, cs)   # keep the callbacks alive

    def last_prove_timings(self):
        names = (ctypes.c_char_p * 20)()
        ms = (ctypes.c_float * 20)()
        k = self._l.tvm_last_prove_timings(self._h, names, ms)
        return [(names[i].decode(), float(ms[i])) for i in range(k)]

    # ---- device-pointer entry points (torch tensors, int64 view of u64, Montgomery) -------
    @staticmethod
    def _dp(t):
        return _vp(t.data_ptr()) if t is not None else None

    def to_mont_(self, t):
        self._chk(self._l.tvm_to_mont_dev(self._h, self._dp(t), t.numel()))
        return t

    def from_mont_(self, t):
        self._chk(self._l.tvm_from_mont_dev(self._h, self._dp(t), t.numel()))
        return t

    def ntt_dev(self, d_in, d_out, d_tmp, log2n, ncols, inverse=False):
        self._chk(self._l.tvm_ntt_bfe_dev(self._h, self._dp(d_in), self._dp(d_out), self._dp(d_tmp), log2n, ncols, int(inverse)))

    def lde_dev(self, d_trace, d_rand, num_rand, log2_trace, log2_cosets, offset, ncols, d_coef, d_out, d_tmp):
        self._chk(self._l.tvm_lde_bfe_dev(self._h, self._dp(d_trace), self._dp(d_rand), num_rand, log2_trace, log2_cosets,
                                          offset, ncols, self._dp(d_coef), self._dp(d_out), self._dp(d_tmp)))

    def hash_rows_dev(self, d_table, col_stride, nrows, ncols, log2_cosets, d_digests):
        self._chk(self._l.tvm_tip5_hash_rows_dev(self._h, self._dp(d_table), col_stride, nrows, ncols, log2_cosets,
                                                 self._dp(d_digests)))

    def air_quotient_dev(self, d_main, main_stride, d_aux, aux_stride, challenges, weights, log2_trace, log2_cosets,
                         offset, d_out, out_stride):
        ch, chp = _np_u64(np.asarray(challenges, dtype=np.uint64).reshape(-1))
        w, wp = _np_u64(np.asarray(weights, dtype=np.uint64).reshape(-1))
        assert ch.size == 189 and w.size == 1812
        self._chk(self._l.tvm_air_quotient_dev(self._h, self._dp(d_main), main_stride, self._dp(d_aux), aux_stride, chp, wp,
                                               log2_trace, log2_cosets, offset, self._dp(d_out), out_stride))

    def merkle_dev(self, d_nodes, nleaves):
        self._chk(self._l.tvm_merkle_build_dev(self._h, self._dp(d_nodes), nleaves))
