"""ctypes binding of libngp_b200.so (the C-ABI declared in include/ngp_b200.h).

The binding is read from the header itself at import, so it cannot drift from what the library was compiled against:
every valued `#define NGP_*` becomes a module constant, every `typedef struct { ... } Ngp*;` a ctypes.Structure of the
same name, and every function declaration an entry of SIGNATURES (name -> (restype, argtypes)). A declaration outside
the rules parse_header states is an import error, never a guess.

There is NO fallback: if the library is missing or a symbol is absent this module raises, and every
operator built on it raises with it. (The CPU oracle under /oracle is test infrastructure and is never
imported from here.)
"""
import ast
import ctypes as C
import operator
import os
import re

from .build import HEADER

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libngp_b200.so")

# C scalar types by value, in parameters, return types and struct fields; any pointer is c_void_p, except a function
# parameter that points to an Ngp* struct, which is POINTER(struct)
_SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint32_t": C.c_uint32, "uint64_t": C.c_uint64,
            "float": C.c_float, "double": C.c_double, "size_t": C.c_size_t, "unsigned long long": C.c_ulonglong}
_OPS = {ast.Add: operator.add, ast.LShift: operator.lshift}
# `type name`, `type* name` or `type name[dim]`
_DECLARATOR = re.compile(r"\s*([\w\s]*\w)(?:\s*(\*+)\s*|\s+)(\w+)\s*(?:\[([^\]]*)\])?\s*")
# the further declarators of a comma list: `name`, `*name` or `name[dim]`
_MORE = re.compile(r"\s*(\*+)?\s*(\w+)\s*(?:\[([^\]]*)\])?\s*")
_STATEMENT = re.compile(r"\s*(?:typedef\s+struct\s*\{([^{}]*)\}\s*(\w+)|([^;{}]+?))\s*;")


def _fail(what, why):
    raise RuntimeError("%s: %s" % (what, why))


def _constant(text, consts, what):
    """value of a #define or array size: integer and float literals, earlier NGP_* names, `+`, `<<` and parentheses"""
    def ev(node):
        if isinstance(node, ast.Constant) and type(node.value) in (int, float):
            return node.value
        if isinstance(node, ast.Name) and node.id in consts:
            return consts[node.id]
        if isinstance(node, ast.BinOp) and type(node.op) in _OPS:
            return _OPS[type(node.op)](ev(node.left), ev(node.right))
        raise ValueError
    try:
        return ev(ast.parse(text.strip(), mode="eval").body)
    except (SyntaxError, ValueError, TypeError):
        _fail(what, "cannot evaluate %r" % text.strip())


def _ctype(base, stars, structs, what, struct_pointers):
    base = " ".join(w for w in base.split() if w != "const")
    if stars:
        return C.POINTER(structs[base]) if struct_pointers and base in structs else C.c_void_p
    if base in _SCALARS:
        return _SCALARS[base]
    if base in structs:
        return structs[base]
    _fail(what, "unsupported type %r" % base)


def _fields(body, structs, consts, name):
    fields = []
    for decl in filter(str.strip, body.split(";")):
        first, *more = decl.split(",")
        m = _DECLARATOR.fullmatch(first)
        if m is None or not all(_MORE.fullmatch(d) for d in more):
            _fail(name, "cannot read the field %r" % " ".join(decl.split()))
        base = m.group(1)
        for stars, field, dim in [m.groups()[1:]] + [_MORE.fullmatch(d).groups() for d in more]:
            what = "%s.%s" % (name, field)
            t = _ctype(base, stars, structs, what, False)
            if dim is not None:
                n = _constant(dim, consts, what)
                if type(n) is not int or n < 1:
                    _fail(what, "array size %r is not a positive integer" % dim)
                t = t * n
            fields.append((field, t))
    return fields


def _function(decl, structs):
    m = re.fullmatch(r"(.*?)\((.*)\)", decl, re.S)
    head = m and _DECLARATOR.fullmatch(m.group(1))
    if not head or head.group(4) is not None:
        _fail(repr(" ".join(decl.split())), "not a function declaration")
    base, stars, name, _ = head.groups()
    args = []
    if m.group(2).strip() != "void":
        for p in m.group(2).split(","):
            a = _DECLARATOR.fullmatch(p)
            if a is None or a.group(4) is not None:
                _fail(name, "cannot read the parameter %r" % " ".join(p.split()))
            args.append(_ctype(a.group(1), a.group(2), structs, name, True))
    return name, (_ctype(base, stars, structs, name, True), args)


def parse_header(path):
    """(constants, structs, signatures) of a C header in include/ngp_b200.h's dialect: `#define NGP_* value`
    (_constant's expressions; a define without a value is skipped), `typedef struct { fields } Ngp*;` (comma lists,
    arrays of constant size, nested structs by value, pointers as c_void_p) and function declarations over _SCALARS,
    pointers and `(void)`. RuntimeError naming the declaration for anything else, and naming the path when the file
    cannot be read."""
    try:
        with open(path) as f:
            src = f.read()
    except OSError as e:
        raise RuntimeError("ngp_pl_b200: cannot read the C header %s: %s" % (path, e))
    try:
        return _parse(src)
    except RuntimeError as e:
        raise RuntimeError("ngp_pl_b200: %s: %s" % (path, e)) from None


def _parse(src):
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    src = re.sub(r"^[ \t]*#[ \t]*ifdef[ \t]+__cplusplus\b.*?^[ \t]*#[ \t]*endif\b", "", src, flags=re.S | re.M)  # extern "C"
    consts = {}
    for name, value in re.findall(r"^[ \t]*#[ \t]*define[ \t]+(\S+)[ \t]*(.*)$", src, re.M):
        if not re.fullmatch(r"NGP_\w+", name):
            _fail("#define " + name, "only NGP_* object-like macros are read")
        if value.strip():
            consts[name] = _constant(value, consts, "#define " + name)
    src = re.sub(r"^[ \t]*#.*$", "", src, flags=re.M)
    structs, signatures = {}, {}
    pos, end = 0, len(src.rstrip())
    while pos < end:
        m = _STATEMENT.match(src, pos)
        if m is None:
            _fail(repr(" ".join(src[pos:].split())[:80]), "not a declaration")
        pos = m.end()
        body, name, decl = m.groups()
        if decl is None:
            structs[name] = type(name, (C.Structure,), {"_fields_": _fields(body, structs, consts, name),
                                                        "__module__": __name__,
                                                        "__doc__": "Mirror of %s in include/ngp_b200.h." % name})
        else:
            fn, sig = _function(decl, structs)
            signatures[fn] = sig
    return consts, structs, signatures


_consts, _structs, SIGNATURES = parse_header(HEADER)
globals().update(_consts)
globals().update(_structs)
ABI_VERSION = _consts["NGP_ABI_VERSION"]
# ngp_render_infer_layout's fields: the NGP_INFER_* indices 0 .. NGP_INFER_LAYOUT_FIELDS - 1, lower-cased, in order
_n_infer = _consts["NGP_INFER_LAYOUT_FIELDS"]
_infer = sorted((v, n[len("NGP_INFER_"):].lower()) for n, v in _consts.items()
                if n.startswith("NGP_INFER_") and 0 <= v < _n_infer)
if [v for v, _ in _infer] != list(range(_n_infer)):
    raise RuntimeError("ngp_pl_b200: %s: the NGP_INFER_* field indices are not 0 .. NGP_INFER_LAYOUT_FIELDS - 1" % HEADER)
NGP_INFER_FIELDS = tuple(n for _, n in _infer)

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "ngp_pl_b200: %s is missing. Build it with `python -m ngp_pl_b200.build` (needs nvcc). "
                "There is no CPU or PyTorch fallback for this path." % LIB_PATH)
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        if h.ngp_abi_version() != ABI_VERSION:
            raise RuntimeError("ngp_pl_b200: ABI version mismatch, rebuild libngp_b200.so")
        _lib = h
    return _lib


def check(rc, what):
    if rc != 0:
        raise RuntimeError("ngp_pl_b200.%s failed with code %d%s" % (
            what, rc, " (invalid argument)" if rc == -22 else " (cudaError_t)"))


def infer_layout(n_rays, max_round_samples):
    """byte offsets of the wavefront's workspace arrays, {field: offset}, and the workspace size"""
    off = (C.c_int64 * len(NGP_INFER_FIELDS))()
    size = lib().ngp_render_infer_layout(int(n_rays), int(max_round_samples), off)
    if size == 0:
        raise ValueError("ngp_render_infer_layout: n_rays and max_round_samples must be >= 1")
    return dict(zip(NGP_INFER_FIELDS, off)), int(size)


def grid_meta(n_levels, log2_hashmap_size, base_resolution, per_level_scale):
    m = _structs["NgpGridMeta"]()
    total = lib().ngp_grid_meta(int(n_levels), int(log2_hashmap_size), int(base_resolution),
                                float(per_level_scale), C.byref(m))
    if total == 0:
        raise RuntimeError("ngp_grid_meta: unsupported grid configuration")
    return m, int(total)
