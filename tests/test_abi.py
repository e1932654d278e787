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
