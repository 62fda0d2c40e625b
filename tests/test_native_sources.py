"""Host plumbing of the CUDA sources has one home: device limits, driver entry points and launch checks live in
csrc/runtime.cu, the split-bf16 stores in csrc/planes.cuh.  A kernel file that grows its own copy fails here."""
import os
import re

CSRC = os.path.join(os.path.dirname(__file__), os.pardir, "slowfast_b200", "csrc")

# (file, function) of the split-bf16 stores kept in place: their loops interleave the split with other work
SPLIT_COPIES_KEPT = {
    ("conv_stem.cu", "stem_input_fold_kernel"),
    ("conv_stem8.cu", "stem8_input_fold_kernel"),
    ("x3d_ops.cu", "dw2_conv_kernel"),
    ("x3d_ops.cu", "dw3_conv_kernel"),
}
RUNTIME_ONLY = re.compile(r"cudaGetDriverEntryPoint|cudaDevAttrMultiProcessorCount|cudaDevAttrMaxSharedMemoryPerBlockOptin|"
                          r"cudaGetLastError|\b148\b")
SPLIT_STORE = re.compile(r"__float2bfloat16_rn\([^;]*-\s*__bfloat162float\(")
DEFINITION = re.compile(r"(\w+)\s*\(")


def _enclosing_function(lines, i):
    """Name of the top-level definition that line i belongs to (the last unindented line that opens one)."""
    for line in reversed(lines[:i + 1]):
        if line[:1].isalpha() or line.startswith("__"):
            names = [n for n in DEFINITION.findall(line) if n != "__launch_bounds__"]
            if names:
                return names[0]
    return None


def test_kernel_files_use_the_shared_runtime_and_split_helpers():
    files = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    assert "runtime.cu" in files and "conv_igemm.cu" in files
    bad, kept = [], set()
    for fn in files:
        lines = open(os.path.join(CSRC, fn)).read().splitlines()
        for i, line in enumerate(lines):
            code = line.split("//")[0]
            if fn != "runtime.cu":
                for m in RUNTIME_ONLY.finditer(line):
                    # the split-K zero fill reports the memset's own error, not a launch
                    if m.group(0) == "cudaGetLastError" and "zero fill of the split-K output" in line:
                        continue
                    bad.append((fn, i + 1, m.group(0)))
            if SPLIT_STORE.search(code):
                where = (fn, _enclosing_function(lines, i))
                if where in SPLIT_COPIES_KEPT:
                    kept.add(where)
                else:
                    bad.append((fn, i + 1, f"split-bf16 store in {where[1]} (use planes.cuh)"))
    assert not bad, bad
    assert kept == SPLIT_COPIES_KEPT, f"stale allow-list entries: {sorted(SPLIT_COPIES_KEPT - kept)}"
