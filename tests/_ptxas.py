"""What ptxas makes of the CUDA sources under parakeet_b200/csrc, without a GPU.  Each source is compiled at most once per pytest
process, with the flags csrc/Makefile builds the library with, and its `ptxas -v` report is parsed into one dict per entry
function.  This is the only module under tests/ that runs nvcc; a test calls it only when nvcc() is not None (needs_nvcc)."""
import concurrent.futures
import functools
import glob
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "parakeet_b200", "csrc")
SOURCES = sorted(os.path.basename(p) for p in glob.glob(os.path.join(CSRC, "*.cu")))
# ptxas remarks that an entry's wgmma.mma_async instructions are serialized, each waiting for the one before: C7510 (the pipeline
# crosses a function call), C7512 (too few registers for the function), C7520 (a dependence on a compiler-inserted
# warpgroup.arrive in a divergent path).  C7519, a warpgroup.arrive injected so a wgmma may use registers, is not serialization.
SERIALIZED = {"C7510", "C7512", "C7520"}


def _make_var(name):
    """The value csrc/Makefile assigns to `name` (`:=` or `?=`)."""
    with open(os.path.join(CSRC, "Makefile")) as f:
        m = re.search(rf"^{name}\s*[:?]=\s*(.+)$", f.read(), re.M)
    assert m, f"csrc/Makefile no longer assigns {name}"
    return m.group(1).strip()


def nvcc():
    """$NVCC, else nvcc on PATH, else the Makefile's default; None when none of them is an executable file."""
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), _make_var("NVCC")):
        if cand and os.path.isfile(cand) and os.access(cand, os.X_OK):
            return cand
    return None


needs_nvcc = pytest.mark.skipif(nvcc() is None, reason="nvcc not available")


def flags():
    """The Makefile's NVCCFLAGS with $(ARCH) expanded: what every object of the library is compiled with."""
    out = _make_var("NVCCFLAGS").replace("$(ARCH)", _make_var("ARCH"))
    assert "$(" not in out, f"unexpanded variable in the Makefile's NVCCFLAGS: {out}"
    return out.split()


def _nvcc(args):
    """Run nvcc with flags() and `args` in csrc/, as make does; -> its stderr, asserting it succeeded."""
    r = subprocess.run([nvcc()] + flags() + args, cwd=CSRC, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"nvcc {' '.join(args)} failed:\n{r.stderr[-4000:]}"
    return r.stderr


def _entries(stderr):
    entries = {}
    for block in stderr.split("Compiling entry function '")[1:]:
        name = block[:block.index("'")]
        props = re.search(rf"Function properties for {re.escape(name)}\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                          r"(\d+) bytes spill loads", block)
        used = re.search(r"Used (\d+) registers.*", block)
        assert props and used, block
        smem = re.search(r"(\d+) bytes smem", used.group(0))
        entries[name] = {"name": name, "registers": int(used.group(1)), "stack": int(props.group(1)),
                         "spill_stores": int(props.group(2)), "spill_loads": int(props.group(3)),
                         "smem": int(smem.group(1)) if smem else 0, "codes": set()}
    for line in stderr.splitlines():
        code = re.search(r"\((C75\d\d)\)", line)
        if code:
            fn = re.search(r"function '([^']+)'", line)
            assert fn and fn.group(1) in entries, f"remark names no entry function: {line}"
            entries[fn.group(1)]["codes"].add(code.group(1))
    return list(entries.values())


@functools.lru_cache(maxsize=None)
def report(source):
    """csrc/<source> compiled with flags() -> {"entries": [...], "stderr": nvcc's stderr}.  An entry is a dict: name (mangled),
    registers, stack (bytes of stack frame), spill_stores, spill_loads (bytes), smem (static shared memory, bytes) and codes, the
    set of C75xx remarks that name the function."""
    with tempfile.TemporaryDirectory(prefix="ptxas-") as d:
        stderr = _nvcc(["-c", source, "-o", os.path.join(d, "out.o")])
    return {"entries": _entries(stderr), "stderr": stderr}


def reports():
    """{source: report(source)} for every .cu under csrc/, compiled concurrently."""
    with concurrent.futures.ThreadPoolExecutor() as pool:
        return dict(zip(SOURCES, pool.map(report, SOURCES)))


def entry(rep, substring):
    """The one entry of a report whose name contains `substring`."""
    hits = [e for e in rep["entries"] if substring in e["name"]]
    assert len(hits) == 1, (substring, [e["name"] for e in hits])
    return hits[0]


@functools.lru_cache(maxsize=None)
def fc_dynamic_smem():
    """pk::fc::kFcSmem, the dynamic shared memory every pwg_layer_fc_kernel launch asks for, printed by a host probe."""
    with tempfile.TemporaryDirectory(prefix="ptxas-") as d:
        probe, exe = os.path.join(d, "probe.cu"), os.path.join(d, "probe")
        with open(probe, "w") as f:
            f.write('#include <stdio.h>\n#include "pwg_fc.cu"\nint main() { printf("%d\\n", pk::fc::kFcSmem); return 0; }\n')
        _nvcc(["-I", CSRC, probe, "pk_common.cu", "-o", exe])
        return int(subprocess.run([exe], check=True, capture_output=True, text=True, timeout=60).stdout)
