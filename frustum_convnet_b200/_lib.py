"""ctypes binding of libfrustum_b200.so (the C ABI declared in include/frustum_b200.h).

The header is the one statement of the ABI; this module reads it once at import:
  - every ``#define FCN_<NAME> <integer>`` becomes the module constant ``<NAME>``;
  - every ``typedef struct { ... } fcn_x;`` becomes ``STRUCTS["fcn_x"]``, a ``ctypes.Structure`` with the fields in
    header order under their C names (every pointer a ``c_void_p``);
  - every ``FCN_API`` prototype becomes a ``SIGNATURES`` entry (restype, argtypes).
Its type table is closed: a construct it does not know (a typedef, bit-field, union, function pointer, nested struct
or unknown type) raises at import and names the declaration, so a new header construct cannot be skipped silently.

No CPU fallback: if the shared library is missing this module raises at load time, and every
entry point raises ``RuntimeError`` with ``fcn_last_error()`` on a non-zero status, mirroring
the reference where AT_ASSERTM / THCudaCheck surface as Python exceptions
(/root/reference/ops/query_depth_point/query_depth_point_cuda.cpp:5-10, ..._kernel.cu:85).
"""
from __future__ import annotations

import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FCN_LIB_PATH") or os.path.join(_HERE, "libfrustum_b200.so")   # override: kernel-variant experiments
HEADER = os.path.join(os.path.dirname(_HERE), "include", "frustum_b200.h")   # FCN_LIB_PATH builds share this tree's header

# The types a field or parameter may have by value.  A pointer may also point to void, char, an fcn_* struct or a
# `struct fcn_*` tag.
SCALARS = {"int": C.c_int, "int32_t": C.c_int, "int64_t": C.c_int64, "uint32_t": C.c_uint32, "uint16_t": C.c_uint16,
           "uint8_t": C.c_uint8, "long long": C.c_longlong, "unsigned long long": C.c_ulonglong, "float": C.c_float, "double": C.c_double,
           "fcn_stream_t": C.c_void_p}
# The header's conditionals as a C compiler sees them.
_CONDITIONS = {"#ifndef FRUSTUM_B200_H_": True, "#if defined(__GNUC__)": True, "#ifdef __cplusplus": False}
_TOKEN = re.compile(r"\w+|\S")
_IDENT = re.compile(r"[A-Za-z_]\w*")


def _preprocess(text):
    """-> ({FCN_NAME: integer}, the C declarations left once comments and directives are gone)."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    defines, lines, active = {}, [], []
    for line in text.splitlines():
        d = " ".join(line.split())
        if not d.startswith("#"):
            if all(active):
                lines.append(line)
        elif d.startswith("#if"):
            if d not in _CONDITIONS:
                raise ValueError("include/frustum_b200.h: unknown conditional %r" % d)
            active.append(_CONDITIONS[d])
        elif d == "#else":
            active[-1] = not active[-1]
        elif d == "#endif":
            active.pop()
        elif all(active) and not (d.startswith("#include ") or d.startswith("#define FCN_API ")
                                  or d == "#define FRUSTUM_B200_H_"):
            m = re.fullmatch(r"#define (FCN_\w+) (-?\d+|\(-?\d+\))", d)
            if not m:
                raise ValueError("include/frustum_b200.h: unknown directive %r" % d)
            defines[m[1]] = int(m[2].strip("()"))
    return defines, "\n".join(lines)


def _declarator(toks, defines, what):
    """Tokens `spec [*...] name [dim]...` -> (spec tokens, pointer depth, name, dims)."""
    dims = []
    while len(toks) >= 3 and toks[-1] == "]" and toks[-3] == "[":
        n = toks[-2]
        if not (n.isdigit() or n in defines):
            raise ValueError("include/frustum_b200.h: unknown dimension %r in %s" % (n, what))
        dims.insert(0, int(n) if n.isdigit() else defines[n])
        toks = toks[:-3]
    if not toks or not _IDENT.fullmatch(toks[-1]):
        raise ValueError("include/frustum_b200.h: cannot read the declarator of %s" % what)
    name, toks, depth = toks[-1], toks[:-1], 0
    while toks and toks[-1] == "*":
        toks, depth = toks[:-1], depth + 1
    return toks, depth, name, dims


def _base(spec, depth, structs, what):
    """The type that specifier tokens name (const dropped), checked against the closed table."""
    base = " ".join(t for t in spec if t != "const")
    if base in SCALARS or base in structs or depth and (base in ("void", "char") or
                                                        re.fullmatch(r"struct fcn_\w+", base)):
        return base
    raise ValueError("include/frustum_b200.h: unknown type %r in %s" % (" ".join(spec), what))


def _type_text(spec, depth):
    return " ".join(spec) + (" " + "*" * depth if depth else "")


def _split(toks, sep):
    out = [[]]
    for t in toks:
        if t == sep:
            out.append([])
        else:
            out[-1].append(t)
    return out


def read_header(text):
    """-> (DEFINES {FCN_NAME: integer}, STRUCTS {fcn_x: ctypes.Structure},
    PROTOTYPES {fcn_f: (return type, [(parameter type, parameter name)])}), the types as C text."""
    defines, body = _preprocess(text)
    decls, level = [[]], 0
    for t in _TOKEN.findall(body):
        level += (t == "{") - (t == "}")
        if t == ";" and level == 0:
            decls.append([])
        else:
            decls[-1].append(t)
    structs, protos = {}, {}
    for d in filter(None, decls):
        what = " ".join(d)
        if d == ["typedef", "void", "*", "fcn_stream_t"]:
            continue
        if d[:2] == ["typedef", "struct"] and "{" in d[2:4] and d[-2] == "}" and _IDENT.fullmatch(d[-1]):
            name, body = d[-1], d[d.index("{") + 1:-2]
            if "{" in body:
                raise ValueError("include/frustum_b200.h: nested struct or union in %s" % name)
            fields = []
            for field in filter(None, _split(body, ";")):
                where, spec = "%s: %s" % (name, " ".join(field)), None
                for piece in _split(field, ","):
                    s, depth, fname, dims = _declarator(piece, defines, where)
                    if spec is None:
                        spec = s
                    elif s:
                        raise ValueError("include/frustum_b200.h: cannot read %s" % where)
                    base = _base(spec, depth, structs, where)
                    t = C.c_void_p if depth else SCALARS.get(base) or structs[base]
                    for n in reversed(dims):
                        t = t * n
                    fields.append((fname, t))
            structs[name] = type(name, (C.Structure,), {"_fields_": fields})
        elif d[:1] == ["FCN_API"] and "(" in d and d[-1] == ")":
            i = d.index("(")
            spec, depth, name, dims = _declarator(d[1:i], defines, what)
            params = d[i + 1:-1]
            if dims or "(" in params or ")" in params:
                raise ValueError("include/frustum_b200.h: cannot read the prototype %s" % what)
            _base(spec, depth, structs, what)
            args = []
            for p in ([] if params == ["void"] else _split(params, ",")):
                s, pdepth, pname, pdims = _declarator(p, defines, what)
                if pdims:
                    raise ValueError("include/frustum_b200.h: array parameter %s in %s" % (pname, name))
                _base(s, pdepth, structs, what)
                args.append((_type_text(s, pdepth), pname))
            protos[name] = (_type_text(spec, depth), args)
        else:
            raise ValueError("include/frustum_b200.h: unknown declaration %s" % what)
    return defines, structs, protos


def param_ctype(text, name, structs):
    """ctypes type of a prototype's parameter or return type, given as C text ("const fcn_group_args *")."""
    spec, depth = text.replace("*", " ").split(), text.count("*")
    base = _base(spec, depth, structs, text)
    if depth == 0 and base in SCALARS:
        return SCALARS[base]
    if depth == 1 and base in structs and spec[0] == "const" and not name.endswith("_dev"):
        return C.POINTER(structs[base])   # the host record an entry reads; a *_dev table is a device address
    if text == "long long *":
        return C.POINTER(C.c_longlong)   # fcn_ipc_export's offset
    if text == "void **":
        return C.POINTER(C.c_void_p)     # fcn_ipc_open's mapped base
    if depth:
        return C.c_void_p
    raise ValueError("include/frustum_b200.h: %s passed by value" % text)


with open(HEADER) as _f:
    DEFINES, STRUCTS, PROTOTYPES = read_header(_f.read())
for _name, _value in DEFINES.items():
    if _name[4:] in globals():
        raise ValueError("include/frustum_b200.h: %s would shadow _lib.%s" % (_name, _name[4:]))
    globals()[_name[4:]] = _value

# name -> (restype, argtypes); kept in one table so tests can check every symbol of the header
SIGNATURES = {name: (C.c_char_p if ret == "const char *" else param_ctype(ret, "", STRUCTS),
                     [param_ctype(t, n, STRUCTS) for t, n in args])
              for name, (ret, args) in PROTOTYPES.items()}

GroupArgs = STRUCTS["fcn_group_args"]
PointnetArgs = STRUCTS["fcn_pointnet_args"]
ConvSeg = STRUCTS["fcn_conv_seg"]
ConvArgs = STRUCTS["fcn_conv_args"]
DecodeOut = STRUCTS["fcn_decode_out"]
MegaSeg = STRUCTS["fcn_mega_seg"]
MegaLayer = STRUCTS["fcn_mega_layer"]
MegaDep = STRUCTS["fcn_mega_dep"]
MegaJob = STRUCTS["fcn_mega_job"]
MegaArgs = STRUCTS["fcn_mega_args"]
TrainSrc = STRUCTS["fcn_train_src"]
TrainSeg = STRUCTS["fcn_train_seg"]
TrainLayer = STRUCTS["fcn_train_layer"]
TrainPool = STRUCTS["fcn_train_pool_args"]
LossArgs = STRUCTS["fcn_loss_args"]
InputArgs = STRUCTS["fcn_input_args"]
DetRecord = STRUCTS["fcn_det_record"]
DetCandidateArgs = STRUCTS["fcn_det_candidate_args"]
DetFinalizeArgs = STRUCTS["fcn_det_finalize_args"]
TrainFrustum = STRUCTS["fcn_train_frustum"]
TrainInputArgs = STRUCTS["fcn_train_input_args"]
ValBatchArgs = STRUCTS["fcn_val_batch_args"]
ValResult = STRUCTS["fcn_val_result"]
KittiEvalArgs = STRUCTS["fcn_kitti_eval_args"]
KittiEvalResult = STRUCTS["fcn_kitti_eval_result"]
SunrgbdEvalArgs = STRUCTS["fcn_sunrgbd_eval_args"]
SunrgbdEvalResult = STRUCTS["fcn_sunrgbd_eval_result"]
FrustumFrame = STRUCTS["fcn_frustum_frame"]
FrustumExtractArgs = STRUCTS["fcn_frustum_extract_args"]
RefineBox = STRUCTS["fcn_refine_box"]
RefineExtractArgs = STRUCTS["fcn_refine_extract_args"]
GtJob = STRUCTS["fcn_gt_job"]
GtExtractArgs = STRUCTS["fcn_gt_extract_args"]
SunrgbdFrame = STRUCTS["fcn_sunrgbd_frame"]
SunrgbdExtractArgs = STRUCTS["fcn_sunrgbd_extract_args"]
DetEvalFeedArgs = STRUCTS["fcn_det_eval_feed_args"]
RefineJobData = STRUCTS["fcn_refine_job_data"]
RefineGtTerms = STRUCTS["fcn_refine_gt_terms"]
RefineJobsArgs = STRUCTS["fcn_refine_jobs_args"]
RefineFrustumTableArgs = STRUCTS["fcn_refine_frustum_table_args"]
FrameExtractArgs = STRUCTS["fcn_frame_extract_args"]
ResampleArgs = STRUCTS["fcn_resample_args"]
FrameRefineArgs = STRUCTS["fcn_frame_refine_args"]
SunrgbdFrameExtractArgs = STRUCTS["fcn_sunrgbd_frame_extract_args"]
SunrgbdDepthArgs = STRUCTS["fcn_sunrgbd_depth_args"]
FrameStoreCursor = STRUCTS["fcn_frame_store_cursor"]
FrameStoreArgs = STRUCTS["fcn_frame_store_args"]

_lib = None


def load():
    """Load (once) and return the ctypes handle.  Raises if the library was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libfrustum_b200.so is missing (%s). Build it with "
                "`python -m frustum_convnet_b200.build` (or __graft_entry__.build()); there is no "
                "CPU or PyTorch fallback for the frustum hot path." % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(status: int, what: str = ""):
    if status != 0:
        msg = load().fcn_last_error().decode(errors="replace")
        raise RuntimeError("libfrustum_b200 %s failed (%d): %s" % (what, status, msg))


def call(name: str, *args):
    check(getattr(load(), name)(*args), name)
