"""ctypes binding of libparakeet_b200.so, derived from its C-ABI header include/parakeet_b200.h.

The header is the one description of the ABI; importing this module parses it once (comments stripped):
  - every `typedef struct ... { ... } NAME;` becomes a ctypes.Structure with the header's field names and order, named NAME
    without its leading `pk_` / `Pk`, CamelCased (pk_conv_gemm_args -> ConvGemmArgs, PkAttentionArgs -> AttentionArgs,
    pk_operand -> Operand); a field of struct type is the nested Structure;
  - every `#define PK_* n` and `enum { PK_* = n }` becomes a module constant (PK_ACT_*, PK_EPI_*, PK_ERR_*);
  - every prototype `<type> pk_*(...)` gets a restype and argtypes, which lib() sets when it first loads the library.
C types map through one closed table: int / int32_t, int64_t, uint32_t, uint64_t and float to the matching ctypes scalar, any
pointer (pk_stream_t included) to c_void_p, a pointer to a header struct to POINTER(that struct) (so C.byref(args) is what a
call passes), a `const char*` return to c_char_p.  Any other spelling raises PkError naming the declaration.

The product path has no CPU fallback: if the shared library is missing or a call fails, an exception is raised.
"""
import ctypes as C
import os
import re
from collections import namedtuple

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libparakeet_b200.so")
HEADER = os.path.join(os.path.dirname(_HERE), "include", "parakeet_b200.h")

WAVEFLOW_TAIL_PARTIALS = 1024      # fp32 scratch elements pk_waveflow_forward_tail needs


class PkError(RuntimeError):
    pass


_SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint32_t": C.c_uint32, "uint64_t": C.c_uint64,
            "float": C.c_float}
_POINTEES = {"void", "char", "double", *_SCALARS}

# params: the header's parameter declarations, as written
Prototype = namedtuple("Prototype", "restype argtypes params")


def _decl(text, what):
    """'const float* const* x' -> ('float', 2, 'x'): one base type, stars and a name; qualifiers are dropped."""
    toks = [t for t in re.findall(r"\w+|\S", text) if t != "const"]
    words = [t for t in toks if t != "*"]
    if len(words) != 2 or toks[0] != words[0] or toks[-1] != words[1] or not all(w.isidentifier() for w in words):
        raise PkError(f"{what}: cannot bind the declaration '{' '.join(text.split())}'")
    return words[0], len(toks) - 2, words[1]


def _ctype(base, stars, structs, what, is_return=False):
    if base == "pk_stream_t" and stars == 0:            # typedef void* pk_stream_t
        return C.c_void_p
    if stars == 0 and base in _SCALARS:
        return _SCALARS[base]
    if stars == 0 and base in structs and not is_return:
        return structs[base]
    if stars == 1 and base in structs:
        return C.POINTER(structs[base])
    if stars > 0 and (base in _POINTEES or base in structs):
        return C.c_char_p if is_return and (base, stars) == ("char", 1) else C.c_void_p
    raise PkError(f"{what}: the C type '{base}{'*' * stars}' has no ctypes mapping in parakeet_b200._lib")


def parse_header(text):
    """(structs {C name: Structure}, prototypes {name: Prototype}, constants {name: int}) declared by a C-ABI header."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    constants = {n: int(v) for n, v in re.findall(r"^\s*#define\s+(PK_\w+)\s+\(?(-?\d+)\)?\s*$", text, flags=re.M)}
    for body in re.findall(r"\benum\s*\{([^}]*)\}", text):
        constants.update((n, int(v)) for n, v in re.findall(r"(PK_\w+)\s*=\s*(-?\d+)", body))
    structs = {}
    for body, cname in re.findall(r"\btypedef\s+struct\s*\w*\s*\{([^}]*)\}\s*(\w+)\s*;", text):
        fields = []
        for stmt in filter(str.strip, body.split(";")):
            first, *more = stmt.split(",")                # `int32_t bmul, hmul` declares two fields
            base = _decl(first, cname)[0]
            for d in [first] + [f"{base} {m}" for m in more]:
                b, stars, name = _decl(d, cname)
                fields.append((name, _ctype(b, stars, structs, f"{cname}.{name}")))
        pyname = "".join(p[:1].upper() + p[1:] for p in re.sub(r"^(pk_|Pk)", "", cname).split("_"))
        structs[cname] = type(pyname, (C.Structure,), {"_fields_": fields})
    prototypes = {}
    for ret, name, params in re.findall(r"^[ \t]*([A-Za-z_][\w \t]*\**)\s*\b(pk_\w+)\s*\(([^)]*)\)\s*;", text, flags=re.M):
        b, stars, _ = _decl(f"{ret} {name}", name)
        decls = [] if params.strip() in ("", "void") else [" ".join(p.split()) for p in params.split(",")]
        argtypes = [_ctype(*_decl(d, name)[:2], structs, name) for d in decls]
        prototypes[name] = Prototype(_ctype(b, stars, structs, name, is_return=True), argtypes, decls)
    return structs, prototypes, constants


with open(HEADER) as _f:
    STRUCTS, PROTOTYPES, _constants = parse_header(_f.read())
globals().update(_constants)
globals().update({cls.__name__: cls for cls in STRUCTS.values()})

_lib = None


def lib():
    """Load (once) and return the ctypes handle, every header prototype's restype and argtypes set; raises PkError when the
    CUDA library has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PkError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name, proto in PROTOTYPES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = proto.restype, proto.argtypes
        _lib = L
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().pk_last_error().decode("utf-8", "replace")
        raise PkError(f"{what} failed with code {rc}: {msg}")


def launch_count():
    return int(lib().pk_launch_count())


def exported_symbols():
    """Names of the entry points include/parakeet_b200.h declares."""
    return sorted(PROTOTYPES)
