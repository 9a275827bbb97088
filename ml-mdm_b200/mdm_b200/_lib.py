"""ctypes binding of libmdm_b200.so (the C ABI declared in include/mdm_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is no fallback:
if the shared object is missing, loading raises, and every compute entry point fails without a GPU.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmdm_b200.so")


class MdmError(RuntimeError):
    pass


class TmapSpec(C.Structure):
    _fields_ = [
        ("ptr", C.c_void_p),
        ("dims", C.c_uint64 * 4),
        ("strides", C.c_uint64 * 4),
        ("box", C.c_uint32 * 4),
    ]


class GemmParams(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("M", C.c_int32),
        ("N", C.c_int32),
        ("K", C.c_int32),
        ("block_n", C.c_int32),
        ("nz1", C.c_int32),
        ("nz2", C.c_int32),
        ("nsplit", C.c_int32),
        ("a_z1_off", C.c_int32),
        ("b_z1_off", C.c_int32),
        ("a_use_z", C.c_int32),
        ("b_use_z", C.c_int32),
        ("H", C.c_int32),
        ("W", C.c_int32),
        ("PW", C.c_int32),
        ("PH", C.c_int32),
        ("tiles_w", C.c_int32),
        ("tiles_h", C.c_int32),
        ("nimg", C.c_int32),
        ("taps", C.c_int32),
        ("flip", C.c_int32),
        ("kblocks_c", C.c_int32),
        ("num_kblocks", C.c_int32),
        ("num_stages", C.c_int32),
        ("alpha", C.c_float),
        ("alpha_dev", C.c_void_p),
        ("bias", C.c_void_p),
        ("residual", C.c_void_p),
        ("out_f32", C.c_void_p),
        ("out_f16", C.c_void_p),
        ("out_act_f16", C.c_void_p),
        ("ldc", C.c_int64),
        ("c_z1_stride", C.c_int64),
        ("c_z2_stride", C.c_int64),
        ("act", C.c_int32),
        ("atomic", C.c_int32),
        ("epi_tma", C.c_int32),
        ("gelu_grad_src", C.c_void_p),
        ("cluster", C.c_int32),
        ("kfactor", C.c_int32),
        ("pair", C.c_int32),
        ("epi_op", C.c_int32),
    ]


_lib = None


def lib():
    """Load (once) and return the ctypes handle. Raises MdmError when the library is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MdmError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). mdm_b200 has no CPU or PyTorch fallback."
            )
        l = C.CDLL(LIB_PATH)
        l.mdm_last_error.restype = C.c_char_p
        l.mdm_launch_count.restype = C.c_ulonglong
        l.mdm_graph_launch_count.restype = C.c_ulonglong
        _lib = l
    return _lib


# void (*mdm_grad_ready_fn)(void* user, void* lo, void* hi)  (include/mdm_b200.h)
GRAD_READY_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p)


def check(rc, what=""):
    if rc != 0:
        msg = lib().mdm_last_error().decode("utf-8", "replace")
        raise MdmError(f"{what} failed (rc={rc}): {msg}")


def launch_count():
    return int(lib().mdm_launch_count())


def graph_launch_count():
    return int(lib().mdm_graph_launch_count())


def tmap(ptr, dims, strides, box):
    s = TmapSpec()
    s.ptr = ptr
    for i in range(4):
        s.dims[i] = int(dims[i])
        s.strides[i] = int(strides[i])
        s.box[i] = int(box[i])
    return s


def gemm_raw(A, B, a_mn, b_mn, params, stream=0):
    check(
        lib().mdm_gemm_raw(C.byref(A), C.byref(B), int(a_mn), int(b_mn), C.byref(params),
                           C.c_void_p(stream)),
        "mdm_gemm_raw",
    )


def gemm_raw_split(A, B, a_mn, b_mn, params, b_lo=0, a_lo=0, stream=0):
    """gemm_raw with second fp16 planes of B and of a K-major A (device pointers, 0 = none): A B + A b_lo + a_lo B."""
    check(
        lib().mdm_gemm_raw_split(C.byref(A), C.byref(B), int(a_mn), int(b_mn), C.byref(params),
                                 C.c_void_p(b_lo or None), C.c_void_p(a_lo or None), C.c_void_p(stream)),
        "mdm_gemm_raw_split",
    )
