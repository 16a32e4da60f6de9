"""ctypes binding of csrc/libgast_b200.so (C ABI: include/gast_b200.h).

The header is the one statement of the ABI: every entry's argument and return types are read from its prototype
when this module is imported, so there is no second copy to keep in step with it.  A parameter or return type
outside the fixed map below raises RuntimeError here, before any call.

There is no fallback: if the shared library is missing or fails to load, importing the
engine raises with the build command.
"""
import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('GAST_B200_LIB') or os.path.join(os.path.dirname(_HERE), 'csrc', 'libgast_b200.so')
# (GAST_B200_LIB: alternative build of the same library, used only for A/B experiments)
HEADER = os.path.join(os.path.dirname(os.path.dirname(_HERE)), 'include', 'gast_b200.h')

GAST_MAX_STAGES = 8
KIND_MODEL, KIND_BLOCK, KIND_LOCAL, KIND_MGLOBAL, KIND_SEMCH, KIND_GLOBAL_HEAD = range(6)

# the C scalar types of the ABI; every pointer (function-pointer typedefs included) is bound as c_void_p
_SCALARS = {'int32_t': C.c_int32, 'int': C.c_int, 'int64_t': C.c_int64, 'uint64_t': C.c_uint64, 'size_t': C.c_size_t,
            'float': C.c_float, 'double': C.c_double}
_RETURNS = dict(_SCALARS, **{'void': None, 'const char*': C.c_char_p})
_PROTOTYPE = re.compile(r'(?P<ret>[\w\s*]+?)\s*\b(?P<name>gast_\w+)\s*\((?P<params>[^()]*)\)')
_PARAM = re.compile(r'(?:const\s+)?(?P<type>\w+)(?P<ptr>(?:\s*\*\s*(?:const\b)?)*)\s*\w*')


def prototypes(text):
    """-> [(name, restype, argtypes)] of every gast_* function the C header `text` declares, in its order.
    RuntimeError names the entry and the type when a parameter or return type has no binding."""
    text = re.sub(r'/\*.*?\*/|//[^\n]*', ' ', text, flags=re.S)
    text = re.sub(r'^\s*#[^\n]*', '', text, flags=re.M)
    fn_pointers = set(re.findall(r'typedef[^;{}]*\(\s*\*\s*(\w+)\s*\)', text))
    out = []
    for stmt in re.split(r'[;{}]', text):
        m = _PROTOTYPE.fullmatch(stmt.strip())
        if m is None:
            continue
        name = m.group('name')
        ret = ' '.join(m.group('ret').replace('*', ' * ').split()).replace(' *', '*')
        if ret not in _RETURNS:
            raise RuntimeError('gast_b200: %s returns %r, which has no ctypes binding' % (name, ret))
        params = [p.strip() for p in m.group('params').split(',')]
        argtypes = []
        for p in ([] if params == ['void'] else params):
            a = _PARAM.fullmatch(p)
            if a is not None and (a.group('ptr') or a.group('type') in fn_pointers):
                argtypes.append(C.c_void_p)
            elif a is not None and a.group('type') in _SCALARS:
                argtypes.append(_SCALARS[a.group('type')])
            else:
                raise RuntimeError('gast_b200: %s takes %r, which has no ctypes binding' % (name, p))
        out.append((name, _RETURNS[ret], argtypes))
    return out


with open(HEADER) as _f:
    _PROTOTYPES = prototypes(_f.read())
SYMBOLS = [name for name, _, _ in _PROTOTYPES]          # every entry the header declares, in its order


class GastCfg(C.Structure):
    _fields_ = [
        ('kind', C.c_int32), ('num_joints', C.c_int32), ('in_features', C.c_int32),
        ('channels', C.c_int32), ('channels_out', C.c_int32), ('num_stages', C.c_int32),
        ('filter_widths', C.c_int32 * GAST_MAX_STAGES),
        ('causal', C.c_int32), ('dense', C.c_int32), ('strided', C.c_int32),
        ('heads', C.c_int32), ('semch_shared_e', C.c_int32), ('semch_bias', C.c_int32),
        ('sym_nnz', C.c_int32), ('con_nnz', C.c_int32),
        ('sym_rows', C.POINTER(C.c_int32)), ('sym_cols', C.POINTER(C.c_int32)),
        ('con_rows', C.POINTER(C.c_int32)), ('con_cols', C.POINTER(C.c_int32)),
        ('device', C.c_int32),
    ]


class GemmAuditSeg(C.Structure):
    """gast_gemm_audit_seg: one K-segment of a GEMM launch's A operand"""
    _fields_ = [('base', C.c_void_p), ('tap_stride', C.c_int64), ('ld', C.c_int32), ('K', C.c_int32),
                ('Kc', C.c_int32), ('T_out', C.c_int32), ('T_in', C.c_int32), ('t_mul', C.c_int32),
                ('t_off', C.c_int32)]


class GemmAudit(C.Structure):
    """gast_gemm_audit: what one GEMM launch receives (gast_debug_set_gemm_audit)"""
    _fields_ = [('index', C.c_int64), ('epi', C.c_int32), ('core', C.c_int32), ('tc_form', C.c_int32),
                ('tma_mask', C.c_int32), ('nseg', C.c_int32), ('seg', GemmAuditSeg * 3), ('W', C.c_void_p),
                ('ldw', C.c_int32), ('N', C.c_int32), ('F', C.c_int32), ('J', C.c_int32), ('fpt', C.c_int32),
                ('ld_out', C.c_int32), ('out', C.c_void_p), ('bias', C.c_void_p), ('relu', C.c_int32),
                ('res_ld', C.c_int32), ('res', C.c_void_p), ('res_T_out', C.c_int32), ('res_T_in', C.c_int32),
                ('res_t_mul', C.c_int32), ('res_t_off', C.c_int32), ('coef', C.c_void_p * 2), ('shift', C.c_void_p),
                ('C', C.c_int32), ('tiles_per_mask', C.c_int32), ('nbr_row_ptr', (C.c_uint8 * 36) * 2),
                ('nbr_col', (C.c_uint8 * 164) * 2), ('ab', C.c_void_p), ('ck', C.c_void_p), ('bg', C.c_void_p),
                ('heads', C.c_int32), ('Cg', C.c_int32)]


GemmAuditFn = C.CFUNCTYPE(C.c_int32, C.c_int32, C.POINTER(GemmAudit), C.c_void_p)


class KernelAudit(C.Structure):
    """gast_kernel_audit: what one expand, row-dot, attention-mix or shrink launch receives
    (gast_debug_set_kernel_audit)"""
    _fields_ = [('index', C.c_int64), ('gemm_index', C.c_int64), ('kind', C.c_int32), ('variant', C.c_int32),
                ('fpb', C.c_int32), ('block', C.c_int32), ('in_type', C.c_int32), ('out_type', C.c_int32),
                ('x', C.c_void_p), ('We', C.c_void_p), ('be', C.c_void_p), ('U', C.c_void_p), ('cab', C.c_void_p),
                ('ab', C.c_void_p), ('Ck', C.c_void_p), ('Ws', C.c_void_p), ('target', C.c_void_p),
                ('loss', C.c_void_p), ('out', C.c_void_p), ('rows', C.c_int64), ('K', C.c_int32), ('ld', C.c_int32),
                ('J', C.c_int32), ('T', C.c_int32), ('T0', C.c_int32), ('stride', C.c_int32), ('taps', C.c_int32),
                ('Fin', C.c_int32), ('heads', C.c_int32), ('Cg', C.c_int32)]


KernelAuditFn = C.CFUNCTYPE(C.c_int32, C.c_int32, C.POINTER(KernelAudit), C.c_void_p)

_lib = None


def load():
    """Load the library once; raise loudly when it is absent (no CPU / torch fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            'gast_b200: %s not found. Build it with `python __graft_entry__.py build` '
            '(or gast-net-3dposeestimation_b200/csrc/build.sh). There is no fallback path.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, restype, argtypes in _PROTOTYPES:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def last_error():
    return load().gast_last_error().decode('utf-8', 'replace')
