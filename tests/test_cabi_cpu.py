"""CPU: the C-ABI library builds, loads and exports every symbol declared in include/*.h
(no compute call is made without a GPU), and the host-side mirror behaves like the reference."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT


def _header_symbols():
    txt = open(os.path.join(ROOT, "include", "frustum_b200.h")).read()
    return sorted(set(re.findall(r"FCN_API\s+[\w\s\*]*?\b(fcn_\w+)\s*\(", txt)))


def test_library_builds_and_exports_every_header_symbol():
    from frustum_convnet_b200 import _lib, build
    build.build()
    lib = _lib.load()
    syms = _header_symbols()
    assert len(syms) >= 10
    for s in syms:
        assert hasattr(lib, s), "missing export " + s
        assert s in _lib.SIGNATURES, "ctypes signature table lacks " + s
    assert set(_lib.SIGNATURES) == set(syms)
    assert lib.fcn_version() >= 100


def test_argument_validation_without_gpu():
    """Validation happens before any CUDA call, so error codes are testable on CPU."""
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    assert lib.fcn_query_depth_point_b3n(1, 4, 4, 0.5, 0, None, None, None, None, None) == -1
    assert b"nsample" in lib.fcn_last_error()
    assert lib.fcn_query_depth_point_b3n(0, 4, 4, 0.5, 4, None, None, None, None, None) == 0  # empty batch
    assert lib.fcn_group_rows(None, None) == -1
    assert lib.fcn_decode_eval(1, 1, 1, 8, 12, 3, None, None, None, None, None, None, None, None, None, None) == -1
    with pytest.raises(RuntimeError):
        _lib.call("fcn_conv_gemm", None, None)
    # rotated-box IoU entry: size / NULL / alignment checks come before the launch
    assert lib.fcn_rbbox_iou_3d_pair(-1, None, None, None, 0.5, None, None) == -1
    assert lib.fcn_rbbox_iou_3d_pair(4, None, None, None, 0.5, None, None) == -1
    assert b"NULL" in lib.fcn_last_error()
    buf = np.zeros(64, dtype=np.float32)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16          # a 16-byte aligned host address
    assert lib.fcn_rbbox_iou_3d_pair(1, base + 4, base, base, 0.5, None, None) == -1
    assert b"aligned" in lib.fcn_last_error()
    assert lib.fcn_rbbox_iou_3d_pair(0, None, None, None, 0.5, None, None) == 0   # nothing to do, no stats


def test_box_iou_wrapper_rejects_cpu_tensors_and_bad_shapes():
    from frustum_convnet_b200.box_iou import rbbox_iou_3d_pair
    with pytest.raises(RuntimeError):
        rbbox_iou_3d_pair(torch.zeros(2, 8, 3), torch.zeros(2, 8, 3))


def test_cpu_tensors_are_rejected_like_the_reference():
    """query_depth_point.py:23-24 asserts .is_cuda; there is no CPU path here either."""
    from frustum_convnet_b200.query_depth_point import QueryDepthPoint
    q = QueryDepthPoint(0.25, 8)
    with pytest.raises(AssertionError):
        q(torch.zeros(1, 3, 16), torch.zeros(1, 3, 4))


def test_state_dict_names_match_reference_layout(golden_loader):
    from frustum_convnet_b200 import config
    for name, modname in (("car_small_b3", "det_base"), ("sunrgbd_full_b2", "det_base_sunrgbd")):
        g, data, sd, w, cfg = golden_loader(name)
        mod = __import__("frustum_convnet_b200." + modname, fromlist=["PointNetDet"])
        m = mod.PointNetDet(3, num_vec=w["num_vec"])
        res = m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
        n = sum(p.numel() for p in m.parameters())
        assert n == (3316777 if modname == "det_base" else 6667589)  # SURVEY.md 8(a7)
        with pytest.raises(RuntimeError):   # eval forward on CPU must fail loudly, not fall back
            m.eval()
            m({k: torch.from_numpy(v) for k, v in data.items()})


def test_engine_weight_pack_is_a_pure_function_of_the_state_dict(golden_loader):
    """BN folding on the host (CPU tensors here): folded 1x1 weights reproduce conv+BN."""
    from frustum_convnet_b200.engine import _fold_bn
    g, data, sd, w, cfg = golden_loader("car_small_b3")
    tsd = {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}
    p = "feat_net.pointnet1.conv1"
    s, sh = _fold_bn(tsd, p + ".1")
    x = torch.randn(5, 3, dtype=torch.float64)
    wq = tsd[p + ".0.weight"].double()[:, :, 0, 0]
    ref = torch.nn.functional.batch_norm(
        (x @ wq.t()).float(), tsd[p + ".1.running_mean"], tsd[p + ".1.running_var"],
        tsd[p + ".1.weight"], tsd[p + ".1.bias"], False, 0.1, 1e-5)
    mine = x @ (wq * s[:, None]).t() + sh
    assert torch.allclose(ref.double(), mine, atol=1e-5)


def test_public_header_is_plain_c(tmp_path):
    """include/frustum_b200.h is the drop-in boundary: it must compile as C99 with nothing but libc headers."""
    import subprocess
    src = tmp_path / "hdr.c"
    src.write_text('#include "frustum_b200.h"\nint main(void) { (void)fcn_version; return 0; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only",
                           "-I", os.path.join(ROOT, "include"), str(src)])
    txt = open(os.path.join(ROOT, "include", "frustum_b200.h")).read()
    includes = re.findall(r'#\s*include\s*[<"]([^>"]+)[>"]', txt)
    assert includes and all(i in ("stdint.h", "stddef.h") for i in includes), includes   # no torch / CUDA headers


def test_ctypes_layout_signatures_and_constants_match_the_compiler(tmp_path):
    """_lib reads its structs, prototypes and constants from include/frustum_b200.h.  A C99 program generated from
    what it read must see, as gcc compiles the header, the same size and alignment of every struct, the same offset
    and size of every field and the same value of every define, and every prototype must have exactly the parameter
    and return types the reader split out of it."""
    import ctypes
    import subprocess
    from frustum_convnet_b200 import _lib
    aliases = {cls.__name__: cls for cls in vars(_lib).values()
               if isinstance(cls, type) and issubclass(cls, ctypes.Structure) and cls is not ctypes.Structure}
    assert aliases == _lib.STRUCTS   # every header struct has its one Python name, and no other class is bound
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "frustum_b200.h"']
    for fn, (ret, args) in _lib.PROTOTYPES.items():
        lines.append('_Static_assert(__builtin_types_compatible_p(__typeof__(&%s), %s (*)(%s)), "%s");'
                     % (fn, ret, ", ".join(t for t, _ in args) or "void", fn))
    lines.append("int main(void) {")
    for name, cls in _lib.STRUCTS.items():
        lines.append('    printf("%s %%zu %%zu\\n", sizeof(%s), _Alignof(%s));' % (name, name, name))
        lines += ['    printf("%s.%s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s *)0)->%s));'
                  % (name, f, name, f, name, f) for f, _ in cls._fields_]
    lines += ['    printf("%s %%lld\\n", (long long)(%s));' % (d, d) for d in _lib.DEFINES]
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines + ["    return 0;", "}", ""]))
    exe = tmp_path / "abi"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)], text=True)
    seen = {k: [int(v) for v in vs] for k, *vs in (ln.split() for ln in out.splitlines())}
    for name, cls in _lib.STRUCTS.items():
        assert seen[name] == [ctypes.sizeof(cls), ctypes.alignment(cls)], name
        for f, _ in cls._fields_:
            assert seen[name + "." + f] == [getattr(cls, f).offset, getattr(cls, f).size], (name, f)
    assert len(_lib.DEFINES) >= 40 and len(_lib.STRUCTS) >= 40 and len(_lib.PROTOTYPES) >= 70
    for d, v in _lib.DEFINES.items():
        assert seen[d] == [v] == [getattr(_lib, d[len("FCN_"):])], d


def test_header_types_map_to_ctypes():
    import ctypes as C
    from frustum_convnet_b200 import _lib
    _, structs, protos = _lib.read_header(
        "#define FCN_N 4\n"
        "typedef void *fcn_stream_t;\n"
        "typedef struct { int first, count; } fcn_b;\n"
        "typedef struct {\n"
        "    const float *w1t, *b1;   /* pointers */\n"
        "    double m[2][FCN_N];\n"
        "    fcn_b dep[FCN_N];\n"
        "    struct fcn_c_ *result;\n"
        "    uint8_t flag;\n"
        "} fcn_a;\n"
        "FCN_API int fcn_f(const fcn_a *args, fcn_stream_t stream);\n")
    assert structs["fcn_a"]._fields_ == [("w1t", C.c_void_p), ("b1", C.c_void_p), ("m", C.c_double * 4 * 2),
                                         ("dep", structs["fcn_b"] * 4), ("result", C.c_void_p), ("flag", C.c_uint8)]
    assert protos == {"fcn_f": ("int", [("const fcn_a *", "args"), ("fcn_stream_t", "stream")])}
    S = _lib.STRUCTS
    for text, name, want in [("int", "n", C.c_int), ("int32_t", "n", C.c_int), ("long long", "n", C.c_longlong),
                             ("unsigned long long", "seed", C.c_ulonglong), ("float", "lr", C.c_float),
                             ("fcn_stream_t", "stream", C.c_void_p), ("const float *", "src", C.c_void_p),
                             ("int64_t *", "idx", C.c_void_p), ("const void *", "handle_64B", C.c_void_p),
                             ("const fcn_group_args *", "args", C.POINTER(S["fcn_group_args"])),
                             ("const fcn_train_layer *", "layers_dev", C.c_void_p),   # a device table
                             ("fcn_val_result *", "result", C.c_void_p),
                             ("long long *", "offset_bytes", C.POINTER(C.c_longlong)),
                             ("void **", "base_out", C.POINTER(C.c_void_p))]:
        assert _lib.param_ctype(text, name, S) is want, text
    for text in ("fcn_group_args", "void", "size_t", "char"):
        with pytest.raises(ValueError):
            _lib.param_ctype(text, "x", S)
    assert _lib.SIGNATURES["fcn_last_error"] == (C.c_char_p, [])


@pytest.mark.parametrize("decl", [
    "typedef struct { size_t n; } fcn_a;",                        # unknown type
    "typedef struct { int n : 3; } fcn_a;",                       # bit-field
    "typedef struct { union { int i; float f; } u; } fcn_a;",     # nested union
    "typedef struct { int (*fn)(int); } fcn_a;",                  # function pointer
    "typedef struct { fcn_b b; } fcn_a;",                         # undeclared struct
    "typedef struct { int x[FCN_NOPE]; } fcn_a;",                 # unknown dimension
    "typedef int fcn_int;",                                       # typedef
    "FCN_API int fcn_f(size_t n, fcn_stream_t stream);",          # unknown parameter type
    "#define FCN_SHIFT (1 << 3)",                                 # non-integer define
])
def test_header_reader_refuses_what_it_does_not_know(decl):
    from frustum_convnet_b200 import _lib
    with pytest.raises(ValueError):
        _lib.read_header("#define FCN_N 4\ntypedef void *fcn_stream_t;\n" + decl + "\n")
