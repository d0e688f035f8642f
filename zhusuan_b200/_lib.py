"""ctypes binding of libzsb200.so (the C ABI declared in include/zsb200.h).

The prototypes are parsed from the header itself, so the Python side cannot
drift from the ABI.  There is NO CPU fallback: if the shared library is
missing, or a compute entry point is reached without CUDA tensors, the call
raises -- it never routes to another implementation.
"""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
LIB_PATH = os.path.join(_HERE, "libzsb200.so")
HEADER_PATH = os.path.join(_ROOT, "include", "zsb200.h")

_CTYPES = {
    "int": ctypes.c_int, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64,
    "uint32_t": ctypes.c_uint32, "int32_t": ctypes.c_int32,
    "float": ctypes.c_float, "size_t": ctypes.c_size_t,
}


def parse_header(path=HEADER_PATH):
    """Return {name: [(ctype, argname, is_host_ptr), ...]} for every
    ``int zsb_*(...)`` prototype in the header."""
    src = open(path).read()
    # keep the /* host */ markers, drop every other comment
    src = re.sub(r"/\*\s*host\s*\*/", " __host__ ", src)
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"\bint\s+(zsb_\w+)\s*\(([^)]*)\)\s*;", src):
        name, args = m.group(1), m.group(2).strip()
        sig = []
        if args and args != "void":
            for a in args.split(","):
                a = a.strip()
                host = "__host__" in a
                a = a.replace("__host__", "").strip()
                is_ptr = "*" in a
                toks = a.replace("*", " ").replace("const", " ").split()
                base, argname = toks[0], toks[-1]
                if is_ptr:
                    if host and base == "int":
                        ct = ctypes.POINTER(ctypes.c_int)
                    elif base == "char":
                        ct = ctypes.c_char_p
                    else:
                        ct = ctypes.c_void_p
                else:
                    ct = _CTYPES[base]
                sig.append((ct, argname, host))
        protos[name] = sig
    return protos


class ZsbError(RuntimeError):
    pass


class _Lib(object):
    def __init__(self):
        self._dll = None
        self.protos = parse_header()

    def load(self):
        if self._dll is None:
            if not os.path.exists(LIB_PATH):
                raise ZsbError(
                    "zhusuan_b200: %s is missing -- build it with "
                    "`python -c 'import __graft_entry__ as g; g.build()'` "
                    "(make -C zhusuan_b200/csrc).  There is no CPU fallback."
                    % LIB_PATH)
            dll = ctypes.CDLL(LIB_PATH)
            for name, sig in self.protos.items():
                fn = getattr(dll, name)     # AttributeError => ABI drift
                fn.restype = ctypes.c_int
                fn.argtypes = [s[0] for s in sig]
            self._dll = dll
        return self._dll

    def last_error(self):
        buf = ctypes.create_string_buffer(512)
        self.load().zsb_last_error(buf, 512)
        return buf.value.decode("utf-8", "replace")

    # kernels launched per successful call (entries that launch two kernels)
    # kernels launched per entry point (default 1): the `gpu_launches` claim of bench.py
    _KERNELS = {"zsb_hmc_mass_stats_f32": 2, "zsb_hmc_dense_traj_prepare_f32": 3, "zsb_hmc_dense_resident_h16_f32": 1, "zsb_sgmcmc_sghmc_f32": 2,
                "zsb_sgmcmc_mean_sq_f32": 2, "zsb_sgmcmc_sgnht_scalar_f32": 2,
                "zsb_split16_pad_f32": 3, "zsb_linear_tc_f32": 2, "zsb_planar_flow_bwd_f32": 2,
                "zsb_iaf_bwd_f32": 2, "zsb_lntm_mstep_grad_f32": 2,
                "zsb_sample_concrete_bwd_f32": 2, "zsb_logprob_concrete_bwd_f32": 2,
                "zsb_gp_cond_bwd_f32": 2, "zsb_conv3x3_wgrad_f32": 2,
                # the tensor-core conv layers' entries, in their common case: a gather-split
                # with its max pass, an activation gradient with the bias sums
                "zsb_conv_gather_split_f32": 3, "zsb_conv_act_grad_f32": 2,
                # the batch-norm entries in training
                "zsb_linear_tc_bn_f32": 3, "zsb_bn_finish_fused_f32": 2, "zsb_bn_grad_f32": 5,
                "zsb_bn_grad_f32out": 3}
    launches = 0

    def call(self, name, *args):
        fn = getattr(self.load(), name)
        rc = fn(*args)
        self.launches += self._KERNELS.get(name, 1)
        if rc != 0:
            raise ZsbError("%s failed (%d): %s" % (name, rc, self.last_error()))
        return rc


lib = _Lib()


def ptr(t):
    """Device pointer of a CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise ZsbError(
            "zhusuan_b200 kernels need CUDA tensors (got a %s tensor); "
            "there is no CPU fallback." % t.device)
    if not t.is_contiguous():
        raise ZsbError("zhusuan_b200: non-contiguous tensor passed to a kernel")
    return t.data_ptr()


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream
