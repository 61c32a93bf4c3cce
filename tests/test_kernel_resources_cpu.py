"""Every entry function of every CUDA source under parakeet_b200/csrc, as ptxas compiles it with the library's own flags, without a
GPU: a 0-byte stack frame, no spills and no serialized wgmma (_ptxas.SERIALIZED), unless EXCEPTIONS names the kernel.  Registers
are not budgeted."""
import _ptxas

pytestmark = _ptxas.needs_nvcc

DEFAULT = {"stack": 0, "spill_stores": 0, "spill_loads": 0, "codes": set()}

# (source, substring of the mangled entry name) -> upper bounds at what ptxas reports for the kernel today (nvcc 12.9), and why
# it exceeds DEFAULT.  A kernel PR that removes a kernel's excess lowers or deletes its row.
EXCEPTIONS = {
    ("conv_gemm.cu", "conv_gemm_kernelILi256E"):
        dict(stack=528, spill_stores=12, spill_loads=60, reason="128 fp32 accumulators per consumer thread under setmaxnreg 232"),
    ("conv_gemm.cu", "conv_gemm_kernelILi128E"): dict(stack=256, reason="a stack frame without spills; not yet traced"),
    ("waveflow_layer.cu", "waveflow_forward_layer_kernelILi128E"):
        dict(stack=304, spill_stores=384, spill_loads=592, codes={"C7512"},
             reason="128 GEMM1 accumulators live with 64 z registers (DESIGN.md section 7)"),
    ("waveflow_layer.cu", "waveflow_flow_kernelILi128E"):
        dict(stack=328, spill_stores=384, spill_loads=592, codes={"C7510"},
             reason="as the forward layer at 128 channels, plus the printf before the dependency-wait trap, a call"),
    ("waveflow_layer.cu", "waveflow_flow_kernelILi64E"):
        dict(stack=24, codes={"C7510"}, reason="the printf before the dependency-wait trap is a call the wgmma pipeline crosses"),
    ("pwg.cu", "pwg_layer_kernel"):
        dict(codes={"C7520"}, reason="the legacy residual layer's wgmma wait on a warpgroup.arrive in a divergent path (DESIGN.md §7)"),
    ("pwg.cu", "pwg_upsample_kernel"): dict(stack=104, reason="per-stage index arrays indexed by the runtime stage count"),
    ("train.cu", "scalar_conv_wgrad_kernel"): dict(stack=64, reason="sw[16] indexed by the runtime tap count"),
    ("fs2.cu", "embed_pe_kernel"): dict(stack=32, reason="the large-argument range reduction of sinf / cosf"),
    ("train.cu", "embed_pe_bwd_kernel"): dict(stack=32, reason="the large-argument range reduction of sinf / cosf"),
}


def test_every_entry_within_its_budget():
    over = []
    for source, rep in _ptxas.reports().items():
        for e in rep["entries"]:
            rows = [row for (src, sub), row in EXCEPTIONS.items() if src == source and sub in e["name"]]
            limit = dict(DEFAULT, **rows[0]) if rows else DEFAULT
            serialized = e["codes"] & _ptxas.SERIALIZED
            if (e["stack"] > limit["stack"] or e["spill_stores"] > limit["spill_stores"] or e["spill_loads"] > limit["spill_loads"]
                    or not serialized <= limit["codes"]):
                over.append(f"{source} {e['name']}: {e['stack']} B stack, {e['spill_stores']} / {e['spill_loads']} B spill stores / "
                            f"loads, serialized {sorted(serialized)}")
    assert not over, "\n".join(over)


def test_every_exception_names_one_entry():
    """A row must not outlive the kernel it was written for: each matches exactly one entry of its source."""
    reps = _ptxas.reports()
    for source, substring in EXCEPTIONS:
        _ptxas.entry(reps[source], substring)
