"""One ownership rule for device memory (DESIGN §3): every device and pinned host buffer of the library is allocated
through a DeviceScope (cb_internal.hpp), which frees it on every exit path. The two exceptions are the context's exchange
region, which CUDA IPC exports and which therefore cannot come from the stream-ordered pool, and the L2 flush buffer,
which stays out of the pool so that flushing before a timed call does not change the pool that call allocates from.
Timing uses scoped events, not events owned by the context."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cilantro_b200", "csrc")
RAW = re.compile(r"\b(cudaMalloc|cudaMallocAsync|cudaFree|cudaFreeAsync|cudaMallocHost|cudaHostAlloc|cudaFreeHost)\(")
# the exchange region (allocated in setup_exchange) and the L2 flush buffer (cb_context_flush_l2), both freed in
# cb_context_destroy
ALLOWED = {"CB_CUDA(cudaMalloc(&ctx->d_xchg, kXchgBytes));", "if (ctx->d_xchg) cudaFree(ctx->d_xchg);",
           "CB_CUDA(cudaMalloc(&ctx->d_flush, ctx->flush_bytes));", "if (ctx->d_flush) cudaFree(ctx->d_flush);"}


def _sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".cpp", ".hpp", ".h")):
            with open(os.path.join(CSRC, name)) as f:
                yield name, f.read()


def test_raw_allocation_calls_only_in_device_scope():
    found = []
    for name, text in _sources():
        if name == "cb_internal.hpp":
            continue
        for no, line in enumerate(text.splitlines(), 1):
            if RAW.search(line) and line.split("//")[0].strip() not in ALLOWED:
                found.append(f"{name}:{no}: {line.strip()}")
    assert not found, "raw allocation calls outside DeviceScope:\n" + "\n".join(found)


def test_exchange_region_and_flush_buffer_are_the_only_exceptions():
    text = dict(_sources())["capi_core.cu"]
    for line in ALLOWED:
        assert text.count(line) == 1, line


def test_context_owns_no_timing_events():
    text = dict(_sources())["cb_internal.hpp"]
    ctx = re.search(r"struct cb_context \{(.*?)\n\};", text, re.S)
    assert ctx, "struct cb_context not found"
    assert not re.search(r"\bev[012]\b", ctx.group(1))
