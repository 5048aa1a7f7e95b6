"""ctypes binding of libt2b200.so (C-ABI declared in include/t2b200.h).

There is deliberately NO CPU / eager fallback: if the shared library is missing or a call fails, the
product path raises. PyTorch is used only for device memory, streams and torch.distributed.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("T2_LIB") or os.path.join(_HERE, "libt2b200.so")     # T2_LIB: experiment builds (tools/)
_lib = None


class T2Error(RuntimeError):
    pass


def load():
    """Load (once) and return the ctypes handle; raises if the extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise T2Error("libt2b200.so is not built: run `python __graft_entry__.py build` "
                          "(there is no CPU fallback for the CUDA hot path)")
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.t2_last_error.restype = ctypes.c_char_p
        _lib.t2_launch_count.restype = ctypes.c_longlong
    return _lib


def check(rc):
    if rc != 0:
        raise T2Error("libt2b200 error %d: %s" % (rc, load().t2_last_error().decode()))


def ptr(t):
    """Device (or host) pointer of a torch tensor as c_void_p; None -> NULL."""
    if t is None:
        return ctypes.c_void_p(0)
    return ctypes.c_void_p(t.data_ptr())


def param_table(info, cfg, n_tensors, trainable=True, base=0):
    """[(name, offset, shape, trainable)] of an engine's flat parameter buffer from its t2_*_param_info function (host-only: no CUDA
    device needed). trainable=False for an info function without the trainable out-parameter (WaveNet): [(name, offset, shape)].
    base is added to every offset."""
    name = ctypes.create_string_buffer(160)
    off, nd, shp, tr = ctypes.c_longlong(), ctypes.c_int(), (ctypes.c_int * 4)(), ctypes.c_int()
    out = []
    for i in range(n_tensors):
        check(info(ctypes.byref(cfg), i, name, 160, ctypes.byref(off), ctypes.byref(nd), shp, *((ctypes.byref(tr),) if trainable else ())))
        t = (name.value.decode(), base + off.value, tuple(shp[k] for k in range(nd.value)))
        out.append(t + (bool(tr.value),) if trainable else t)
    return out


def adam_scratch_floats(n_tensors, n_total):
    """fp32 elements of t2_adam_step's d_scratch: per-tensor norms, the global norm and one partial per tensor segment of a 4096-element
    chunk (include/t2b200.h)"""
    return 2 * n_tensors + (n_total + 4095) // 4096


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- mirrors of the engine-level test structs of include/t2b200.h (t2_dbg_act_gemm / t2_dbg_wgrad_tiles) ----
class DbgAct(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_void_p), ("C", ctypes.c_int), ("T", ctypes.c_int), ("B", ctypes.c_int), ("L", ctypes.c_int),
                ("ld", ctypes.c_int)]


class DbgSeg(ctypes.Structure):
    _fields_ = [("map", ctypes.c_int), ("shift", ctypes.c_int), ("k0", ctypes.c_int), ("nkb", ctypes.c_int),
                ("layer0", ctypes.c_int), ("nlayers", ctypes.c_int)]


class DbgGemm(ctypes.Structure):
    _fields_ = [("a", DbgAct * 4), ("na", ctypes.c_int),
                ("seg", DbgSeg * 16), ("nseg", ctypes.c_int),
                ("w", ctypes.c_void_p), ("wN", ctypes.c_int), ("wK", ctypes.c_int), ("wL", ctypes.c_int),
                ("w_layer", ctypes.c_int), ("w_k0", ctypes.c_int),
                ("T", ctypes.c_int), ("B", ctypes.c_int), ("n_tiles", ctypes.c_int), ("ksplit", ctypes.c_int),
                ("epi", ctypes.c_int), ("BN", ctypes.c_int), ("cluster", ctypes.c_int), ("cluster_used", ctypes.c_int),
                ("ptr", ctypes.c_void_p * 12), ("f", ctypes.c_float * 6), ("i", ctypes.c_int * 12), ("seed", ctypes.c_ulonglong)]


class DbgWgradTile(ctypes.Structure):
    _fields_ = [("a_map", ctypes.c_int), ("a_ch0", ctypes.c_int), ("a_shift", ctypes.c_int), ("a_layer", ctypes.c_int),
                ("b_map", ctypes.c_int), ("b_ch0", ctypes.c_int), ("b_shift", ctypes.c_int), ("b_layer", ctypes.c_int),
                ("out_off", ctypes.c_longlong), ("ldc", ctypes.c_int), ("m_valid", ctypes.c_int), ("n_valid", ctypes.c_int),
                ("scale", ctypes.c_float), ("accumulate", ctypes.c_int), ("div", ctypes.c_void_p)]


class DbgKernel(ctypes.Structure):
    """t2_dbg_kernel_t: one Tacotron / CBHG kernel launch for t2_dbg_taco_kernel / t2_dbg_cbhg_kernel"""
    _fields_ = [("kernel", ctypes.c_int), ("p", ctypes.c_void_p * 16), ("i", ctypes.c_longlong * 16), ("f", ctypes.c_float * 4),
                ("seed", ctypes.c_ulonglong), ("step", ctypes.c_void_p)]
