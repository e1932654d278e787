"""CPU tests: every kernel of the device library is launched through dp_launch / dp_launch_cluster (common.cuh), which count the
launch for dp_kernel_launches and return its error; the per-thread context takes no lock; and every completion word a kernel
writes for the host goes through dp_publish (a system-scope fence, then the volatile store)."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deep-prove_b200", "csrc")
HELPERS = ("dp_launch", "dp_launch_cluster")

# __threadfence_system() outside dp_publish, by file and the statement that follows it
FENCES = {
    ("sumcheck.cu", "u32 t = atomicAdd(done, 1u)"):
        "sc_signal: orders the block's message stores before its ticket; the last block publishes through dp_publish",
    ("sumcheck.cu", "c0 = chal[1]"):
        "the resident kernel's mailbox read: a fence before loading the challenge the host posted, not a publish",
}


def strip_comments(src):
    """the source with its comments blanked out (string and character literals kept; offsets and line numbers unchanged)"""
    tok = re.compile(r'"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'|//[^\n]*|/\*.*?\*/', re.S)
    return tok.sub(lambda m: m.group(0) if m.group(0)[0] in "\"'" else re.sub(r"[^\n]", " ", m.group(0)), src)


def sources():
    paths = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")))
    assert any(p.endswith("common.cuh") for p in paths) and len(paths) >= 8, "csrc/ not found or incomplete"
    return {os.path.basename(p): strip_comments(open(p).read()) for p in paths}


def body_span(src, signature):
    """(start, end) of the braces of the function whose definition matches `signature`"""
    m = re.search(signature, src)
    assert m, "definition not found: " + signature
    i = src.index("{", m.end())
    depth = 0
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return i, j + 1
    raise AssertionError("unbalanced braces after " + signature)


def outside(spans, pos):
    return all(not (a <= pos < b) for a, b in spans)


def where(name, src, pos):
    return "%s:%d" % (name, src.count("\n", 0, pos) + 1)


def test_every_launch_goes_through_the_helpers():
    srcs = sources()
    common = srcs["common.cuh"]
    spans = [body_span(common, r"cudaError_t\s+%s\s*\(" % h) for h in HELPERS]
    bad = []
    for name, src in srcs.items():
        for m in re.finditer(r"<<<|\bcudaLaunchKernelEx\b|\bdp_count_launch\s*\(", src):
            if name == "common.cuh" and not outside(spans, m.start()):
                continue
            line = src[src.rfind("\n", 0, m.start()) + 1:src.find("\n", m.start())]
            if m.group(0).startswith("dp_count_launch") and re.match(r"\s*void\s+dp_count_launch\s*\(\s*\)", line):
                continue   # its declaration (common.cuh) and definition (context.cu)
            bad.append("%s: %s" % (where(name, src, m.start()), line.strip()))
    assert bad == [], "launches or launch counts outside dp_launch / dp_launch_cluster:\n" + "\n".join(bad)
    for h in HELPERS:
        body = common[slice(*spans[HELPERS.index(h)])]
        assert "dp_count_launch()" in body and "cudaGetLastError()" in body, h + " must count the launch and return its error"


def test_no_launch_counting_macro_and_no_lock_on_the_context():
    for name, src in sources().items():
        for word in ("DP_LAUNCHED", "recursive_mutex"):
            assert word not in src, "%s still uses %s" % (name, word)


def test_completion_words_are_published_through_dp_publish():
    srcs = sources()
    common = srcs["common.cuh"]
    publish = body_span(common, r"void\s+dp_publish\s*\(")
    seen = set()
    bad = []
    for name, src in srcs.items():
        for m in re.finditer(r"__threadfence_system\s*\(\s*\)\s*;", src):
            if name == "common.cuh" and not outside([publish], m.start()):
                continue
            nxt = " ".join(src[m.end():src.index(";", m.end())].split())
            if (name, nxt) in FENCES:
                seen.add((name, nxt))
            else:
                bad.append("%s: __threadfence_system(); %s;" % (where(name, src, m.start()), nxt))
    assert bad == [], "a system fence outside dp_publish (publish a completion word with dp_publish, or list the fence here):\n" + "\n".join(bad)
    assert seen == set(FENCES), "listed fences that no longer exist: %s" % sorted(set(FENCES) - seen)
    assert sum(src.count("dp_publish(") for src in srcs.values()) >= 8
