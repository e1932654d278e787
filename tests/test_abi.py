"""CPU tests: the C-ABI library loads, exports every symbol include/deepprove_b200.h declares (and the host
library imports no other), and refuses to compute without a GPU (no CPU fallback)."""
import os
import re
import subprocess
import dpb200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "deepprove_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dp_[a-z0-9_]+)\s*\(", src)))


def test_every_declared_symbol_is_exported():
    lib = dpb200.lib()
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), "libdeepprove_b200.so does not export %s" % s
    assert sorted(dpb200.ABI_SYMBOLS) == syms, "dpb200.ABI_SYMBOLS out of sync with the header"


def test_host_library_links_only_against_the_c_abi():
    """libdeepprove_host.so calls into libdeepprove_b200.so through the public header alone (DESIGN.md section 1)"""
    dpb200.host()
    out = subprocess.run(["nm", "-D", "--undefined-only", dpb200.HOST_LIB_PATH], check=True, capture_output=True, text=True).stdout
    imported = set(re.findall(r"\bU (dp_[a-z0-9_]+)\b", out))
    assert imported, "no dp_* import found: nm output not understood"
    assert sorted(imported - set(header_symbols())) == []


def test_no_cpu_fallback_without_gpu():
    lib = dpb200.lib()
    if lib.dp_device_count() > 0:
        return  # on the GPU box this is covered by the gpu tests
    assert lib.dp_init(0) == dpb200.DP_ERR_NO_DEVICE
    assert b"no CPU fallback" in lib.dp_last_error()
    import ctypes as C
    import numpy as np
    a = np.arange(8, dtype=np.uint64)
    h = C.c_void_p()
    assert lib.dp_mle_upload(a.ctypes.data_as(C.c_void_p), 8, 0, C.byref(h)) == dpb200.DP_ERR_NO_DEVICE


def test_product_does_not_reference_oracle():
    """the shipped path must not import, link or execute oracle/"""
    pkg = os.path.join(ROOT, "deep-prove_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".cu", ".cuh", ".cpp", ".hpp", ".py", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "oracle/" not in txt.replace("Never imports anything from oracle/", "").replace("Nothing here touches oracle/", "") \
                    and "oracle_py" not in txt and "libdp_oracle" not in txt, f


def test_wait_mode_switch_needs_no_device():
    """dp_set_wait_mode / dp_get_wait_mode (how proving threads wait for the device: spin, or sleep on the library's poller) are plain
    process-wide settings: usable before dp_init and without a GPU; an unknown mode is refused"""
    lib = dpb200.lib()
    before = lib.dp_get_wait_mode()
    try:
        assert lib.dp_set_wait_mode(1) == 0 and lib.dp_get_wait_mode() == 1
        assert lib.dp_set_wait_mode(0) == 0 and lib.dp_get_wait_mode() == 0
        assert lib.dp_set_wait_mode(7) == dpb200.DP_ERR_INVALID
    finally:
        lib.dp_set_wait_mode(before)


def test_sharded_commit_refuses_without_gpu_and_bad_worlds():
    lib = dpb200.lib()
    if lib.dp_device_count() > 0:
        return
    import ctypes as C
    h = C.c_void_p()
    assert lib.dp_pcs_commit_shard(None, 20, 0, 2, C.byref(h)) == dpb200.DP_ERR_NO_DEVICE


# ---- the ctypes signature table (dpb200.SIGNATURES) against the C declarations ------------------------------------------------
def _c_prototypes(path, prefix, end):
    """{name: (return declaration, [argument declarations])} of every function `prefix*` declared (end ";") or defined (end "{")"""
    src = open(os.path.join(ROOT, path)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    src = re.sub(r"^\s*#[^\n]*", "", src, flags=re.M)
    out = {}
    for m in re.finditer(r"\b(%s\w+)\s*\(" % prefix, src):
        i, depth = m.end(), 1
        while depth:                                   # the matching parenthesis: arguments like `char (*names)[64]` nest
            depth += {"(": 1, ")": -1}.get(src[i], 0)
            i += 1
        if src[i:].lstrip()[:1] != end:
            continue                                   # a call, or a forward declaration in a .cpp
        args, depth, cur = [], 0, ""
        for ch in src[m.end():i - 1]:
            depth += {"(": 1, ")": -1}.get(ch, 0)
            if ch == "," and depth == 0:
                args.append(cur.strip()); cur = ""
            else:
                cur += ch
        args.append(cur.strip())
        ret = re.split(r"[;{}]", src[:m.start()])[-1].replace('extern "C"', "").strip()
        out[m.group(1)] = (ret, [a for a in args if a not in ("", "void")])
    return out


def _c_class(decl):
    """pointer / 64-bit integer / 32-bit integer / double / void, from a C declaration"""
    if "*" in decl or "[" in decl or "::Fn" in decl:
        return "pointer"
    base = decl.replace("const ", "").split()[0]
    return {"uint64_t": "i64", "int64_t": "i64", "uint32_t": "i32", "int": "i32", "double": "double", "void": "void"}[base]


def _ctypes_class(t):
    import ctypes as C
    return {C.c_void_p: "pointer", C.c_char_p: "pointer", C.c_uint64: "i64", C.c_int64: "i64", C.c_uint32: "i32", C.c_int: "i32",
            C.c_double: "double", None: "void"}[t]


def test_signature_table_matches_the_c_declarations():
    """every entry point of include/deepprove_b200.h and host/capi.cpp has a table entry with its argument count and, argument by
    argument and for the return value, its class; every dph_* symbol the host library exports is in the table and every table entry
    is exported by its library"""
    declared = dict(_c_prototypes("include/deepprove_b200.h", "dp_", ";"))
    defined = _c_prototypes("deep-prove_b200/host/capi.cpp", "dph_", "{")
    assert len(declared) >= 80 and len(defined) >= 25, "prototypes not found: parser out of date"
    declared.update(defined)
    table = dpb200.SIGNATURES
    for name, (ret, args) in declared.items():
        assert name in table, "%s has no ctypes signature" % name
        res, argtypes = table[name]
        assert len(argtypes) == len(args), name
        assert [_ctypes_class(t) for t in argtypes] == [_c_class(a) for a in args], name
        assert _ctypes_class(res) == _c_class(ret + (" x" if ret.endswith("*") else "")), name
    assert set(table) - set(declared) == set(dpb200.TEST_HOOKS)
    out = subprocess.run(["nm", "-D", "--defined-only", dpb200.HOST_LIB_PATH], check=True, capture_output=True, text=True).stdout
    exported = set(re.findall(r"\b(dph_[a-z0-9_]+)\b", out))
    assert exported == {n for n in table if n.startswith("dph_")}
    lib, host = dpb200.lib(), dpb200.host()
    for name in table:
        assert hasattr(host if name.startswith("dph_") else lib, name), "%s is not exported" % name


def test_signatures_are_declared_only_in_the_table():
    """no .argtypes / .restype assignment on a function of the two libraries outside dpb200.py"""
    found = []
    for d in ("deep-prove_b200", "tests", "tools"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, d)):
            for f in files:
                path = os.path.join(dirpath, f)
                if not f.endswith(".py") or path == os.path.abspath(dpb200.__file__):
                    continue
                for line in open(path):
                    if re.search(r"\.(argtypes|restype)\s*=", line) and set(re.findall(r"\bdph?_\w+", line)) & set(dpb200.SIGNATURES):
                        found.append("%s: %s" % (f, line.strip()))
    assert found == []
