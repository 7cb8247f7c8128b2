"""CPU tests of the drop-in boundary: the C-ABI library loads, exports every symbol include/rpk.h
declares, and refuses to run without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

import rpk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_source():
    """include/rpk.h without comments and preprocessor lines, whitespace collapsed (multi-line declarations joined)"""
    src = open(os.path.join(ROOT, "include", "rpk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
    return " ".join(src.split())


def header_symbols():
    return sorted(set(re.findall(r"\b(rpk_[a-z0-9_]+)\s*\(", header_source())))


def header_prototypes():
    """-> {name: (return type, [parameter declarations])}"""
    protos = {}
    for ret, name, params in re.findall(r"(?:^|(?<=[;{}]))\s*([A-Za-z_][\w\s*]*?)\s*\b(rpk_\w+)\s*\(([^()]*)\)\s*;", header_source()):
        params = [p.strip() for p in params.split(",")]
        protos[name] = (ret.strip(), [] if params == ["void"] else params)
    return protos


# C scalar type -> (kind, bytes, signed)
C_SCALARS = {"int": ("int", 4, True), "unsigned": ("int", 4, False), "int32_t": ("int", 4, True), "uint32_t": ("int", 4, False),
             "uint64_t": ("int", 8, False), "size_t": ("int", C.sizeof(C.c_size_t), False), "float": ("float", 4, True)}


def c_sig(decl: str, is_param: bool):
    """C type of a parameter declaration (with its name) or of a return type -> "void", "pointer" or a C_SCALARS entry"""
    if "*" in decl or "[" in decl:
        return "pointer"
    words = [w for w in decl.split() if w != "const"]
    if is_param:
        words = words[:-1]
    return "void" if words == ["void"] else C_SCALARS[" ".join(words)]


def ctypes_sig(t):
    if t is None:
        return "void"
    if t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer):
        return "pointer"
    if t in (C.c_float, C.c_double):
        return ("float", C.sizeof(t), True)
    return ("int", C.sizeof(t), t(-1).value < 0)


def test_library_exports_every_declared_symbol():
    lib = rpk._ffi.load()
    declared = header_symbols()
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/rpk.h but not exported by librpk.so"
    assert sorted(rpk._ffi.SYMBOLS) == declared, "python binding out of sync with include/rpk.h"


def test_binding_types_match_the_header():
    """Every ctypes declaration has the header's parameter count, and each parameter and return value its C type's kind
    (pointer or scalar), width and signedness: a size_t declared 32-bit or a uint32_t declared signed would truncate or
    sign-extend silently.  RpkStats has rpk_stats's fields, in order, with their types."""
    protos = header_prototypes()
    assert sorted(protos) == header_symbols()
    for name, (restype, argtypes) in rpk._ffi.ABI.items():
        ret, params = protos[name]
        assert len(argtypes) == len(params), f"{name}: {len(argtypes)} argtypes for {len(params)} parameters"
        for i, (t, p) in enumerate(zip(argtypes, params)):
            assert ctypes_sig(t) == c_sig(p, True), f"{name} parameter {i} `{p}` declared as {t.__name__}"
        assert ctypes_sig(restype) == c_sig(ret, False), f"{name}: returns `{ret}`, restype {restype}"

    body = re.search(r"typedef struct rpk_stats \{(.*?)\} rpk_stats;", header_source()).group(1)
    fields = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        ctype, names = decl.split(None, 1)
        fields += [(n.strip(), C_SCALARS[ctype]) for n in names.split(",")]
    assert [(n, ctypes_sig(t)) for n, t in rpk._ffi.RpkStats._fields_] == fields


def test_abi_version_and_null_handling():
    lib = rpk._ffi.load()
    assert lib.rpk_abi_version() == 2
    lib.rpk_destroy(None)  # no-op
    assert lib.rpk_launch_count(None) == 0
    assert lib.rpk_offers_upload(None, 0, None, None, None, None, None, None) == rpk._ffi.RPK_EINVAL
    assert lib.rpk_create(0, None, C.byref(C.c_void_p())) == rpk._ffi.RPK_EINVAL
    assert lib.rpk_create(9, None, C.byref(C.c_void_p())) == rpk._ffi.RPK_EINVAL
    assert b"n_gpus" in lib.rpk_last_error(None)


def test_no_cpu_fallback_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present; this test pins the behaviour of the CPU-only box")
    with pytest.raises(rpk.RpkError) as ei:
        rpk.Engine(1)
    assert ei.value.code == rpk._ffi.RPK_ENODEV
    assert "no CPU fallback" in str(ei.value)


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under the package or include/ may mention it."""
    pkg = os.path.join(ROOT, "k8s-runpod-kubelet_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cc", ".cpp", ".hpp", ".go")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle" not in txt.lower(), os.path.join(dirpath, f)


def test_header_is_plain_c(tmp_path):
    """include/rpk.h must be bindable from cgo: it has to compile as C99 on its own, with no C++ or CUDA types."""
    import subprocess

    src = tmp_path / "use_rpk.c"
    src.write_text('#include "rpk.h"\nint main(void) { rpk_ctx* c = 0; rpk_stats s; (void)s; return rpk_create(1, 0, &c) == RPK_ENODEV ? 0 : 0; }\n')
    out = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


def test_c_program_links_against_librpk(tmp_path):
    """A C caller (what cgo generates) links against librpk.so and gets RPK_ENODEV / a ctx, never a crash."""
    import subprocess

    src = tmp_path / "link_rpk.c"
    src.write_text('#include <stdio.h>\n#include "rpk.h"\nint main(void) { rpk_ctx* c = 0; int rc = rpk_create(1, 0, &c);\n'
                   ' printf("%d %d %s\\n", rpk_abi_version(), rc, rc ? rpk_last_error(0) : "ok"); if (c) rpk_destroy(c); return 0; }\n')
    exe = tmp_path / "link_rpk"
    libdir = os.path.join(ROOT, "k8s-runpod-kubelet_b200", "lib")
    out = subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", libdir, "-lrpk",
                          f"-Wl,-rpath,{libdir}"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0, run.stderr
    ver, rc = run.stdout.split()[:2]
    assert ver == "2" and int(rc) in (0, rpk._ffi.RPK_ENODEV)
