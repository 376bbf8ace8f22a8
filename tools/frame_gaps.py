"""Where the device idles inside one frame: every kernel, memset and copy a warm sync-free
`render_device` frame puts on the render stream, with its start and end, the idle time before it,
and the event records (the renderer's stage and sort-pass timing events) between them, taken
from a `torch.profiler` trace with CUDA activities. The sum of the idle time between the frame's
first and last event record (the renderer's ev[0] .. ev[6]) is the fixed cost of the chain's
step boundaries.

A second part answers whether an event record between two kernels keeps the second from being
launched early under programmatic dependent launch: chains of two short kernels, launched plainly,
with the programmatic-serialization attribute, and with the attribute and a `cudaEventRecord` of
an event created with `cudaEventDisableTiming` between every pair; the host queues each chain behind a kernel that holds the stream, so that the
chain is timed on the device alone. The probe is compiled with nvcc into a temporary directory.

Prints the card and its power limit from the same run.

    python tools/frame_gaps.py [--workload paris4k] [--frames 6] [--pdl 0|1] [--no-probe] [--trace out.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

PROBE_SRC = r"""
#include <cuda_runtime.h>
__device__ __forceinline__ void wait_prior() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void let_next() { asm volatile("griddepcontrol.launch_dependents;" :::); }
// One short step of a chain: every CTA reads what the step before wrote and writes its own slot.
__global__ void step_kernel(const unsigned* in, unsigned* out, int n) {
    let_next();
    wait_prior();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[(i * 7) % n] + 1u;
}
// Holds the stream while the host queues the chain, so that the chain is timed on the device alone.
__global__ void hold_kernel(long long cycles) {
    const long long t0 = clock64();
    while (clock64() - t0 < cycles) {}
}
static cudaError_t launch(bool pdl, cudaStream_t s, const unsigned* in, unsigned* out, int n) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((n + 255) / 256);
    cfg.blockDim = dim3(256);
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, step_kernel, in, out, n);
}
// Microseconds per kernel of a chain of 2 * pairs kernels. mode 0: plain launches; 1: every kernel
// with programmatic stream serialization; 2: as 1 with an event record between the two kernels of
// every pair. Negative on a CUDA error.
extern "C" double probe(int mode, int pairs, int n) {
    cudaStream_t s;
    unsigned *a, *b;
    cudaEvent_t e0, e1, mid;
    if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) || cudaMalloc(&a, n * 4) || cudaMalloc(&b, n * 4) ||
        cudaEventCreate(&e0) || cudaEventCreate(&e1) || cudaEventCreateWithFlags(&mid, cudaEventDisableTiming))
        return -1.0;
    cudaMemsetAsync(a, 0, n * 4, s);
    cudaMemsetAsync(b, 0, n * 4, s);
    for (int rep = 0; rep < 2; ++rep) {  // rep 0 warms up
        hold_kernel<<<1, 1, 0, s>>>(40000000ll);  // ~20 ms
        cudaEventRecord(e0, s);
        for (int p = 0; p < pairs; ++p) {
            launch(mode > 0, s, a, b, n);
            if (mode == 2) cudaEventRecord(mid, s);
            launch(mode > 0, s, b, a, n);
        }
        cudaEventRecord(e1, s);
    }
    float ms = 0.0f;
    cudaError_t err = cudaStreamSynchronize(s);
    cudaEventElapsedTime(&ms, e0, e1);
    cudaFree(a);
    cudaFree(b);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaEventDestroy(mid);
    cudaStreamDestroy(s);
    return err == cudaSuccess ? 1000.0 * ms / (2.0 * pairs) : -1.0;
}
"""


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    import torch
    return out or torch.cuda.get_device_name(0)


def run_probe(pairs=400, n=132 * 4 * 256):
    """Microseconds per kernel of the three chains (see PROBE_SRC), in alternating rounds."""
    with tempfile.TemporaryDirectory() as tmp:
        src, lib = os.path.join(tmp, "probe.cu"), os.path.join(tmp, "probe.so")
        with open(src, "w") as f:
            f.write(PROBE_SRC)
        nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
        subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-shared", "-Xcompiler", "-fPIC",
                               "-o", lib, src])
        dll = C.CDLL(lib)
        dll.probe.restype = C.c_double
        dll.probe.argtypes = [C.c_int, C.c_int, C.c_int]
        res = {0: [], 1: [], 2: []}
        for _ in range(3):
            for mode in (0, 1, 2):
                res[mode].append(dll.probe(mode, pairs, n))
    return res


def frame_ops(trace_path, label):
    """The render-stream ops and event records of the last range named `label`, in stream order."""
    with open(trace_path) as f:
        evs = json.load(f)["traceEvents"]
    frames = [e for e in evs if e.get("name") == label and e.get("ph") == "X" and e.get("cat") == "user_annotation"]
    last = max(frames, key=lambda e: e["ts"])
    t0, t1, tid = last["ts"], last["ts"] + last["dur"], last["tid"]
    runtime = sorted((e for e in evs if e.get("cat") == "cuda_runtime" and e.get("ph") == "X" and e.get("tid") == tid
                      and t0 <= e["ts"] <= t1), key=lambda e: e["ts"])
    gpu = {}
    for e in evs:
        if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy"):
            gpu[e["args"].get("correlation")] = e
    ops, stream = [], None
    for r in runtime:
        g = gpu.get(r["args"].get("correlation"))
        if g is not None:
            stream = stream if stream is not None else g["args"].get("stream")
            ops.append(("op", g))
        elif r["name"].startswith("cudaEventRecord"):
            ops.append(("event", r))
    return [(k, e) for k, e in ops if k == "event" or e["args"].get("stream") == stream]


def report(ops):
    """Prints the table and returns the idle microseconds between the first and last event record."""
    marks = [i for i, (k, _) in enumerate(ops) if k == "event"]
    lo, hi = (marks[0], marks[-1]) if marks else (0, len(ops))
    base = next((e["ts"] for k, e in ops if k == "op"), 0.0)
    print(f"{'start_us':>10} {'end_us':>10} {'dur_us':>8} {'idle_us':>8}  name")
    prev_end, idle, n_ev, boundaries = None, 0.0, 0, []
    for i, (k, e) in enumerate(ops):
        if k == "event":
            print(f"{'':>10} {'':>10} {'':>8} {'':>8}  -- event record #{n_ev}")
            n_ev += 1
            continue
        s, d = e["ts"] - base, e["dur"]
        gap = None if prev_end is None else s - prev_end
        inside = lo < i < hi and gap is not None
        if inside:
            idle += max(gap, 0.0)
            boundaries.append((gap, e["name"][:60]))
        print(f"{s:10.1f} {s + d:10.1f} {d:8.1f} {'' if gap is None else f'{gap:8.1f}'}  {e['name'][:90]}")
        prev_end = s + d
    return idle, boundaries


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="paris4k")
    ap.add_argument("--frames", type=int, default=6)
    ap.add_argument("--pdl", type=int, default=None, help="the library's pdl option (default: as built / FORMA_PDL)")
    ap.add_argument("--no-probe", action="store_true")
    ap.add_argument("--trace", default=None, help="also keep the chrome trace here")
    args = ap.parse_args(argv)
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function

    import forma_b200
    from forma_b200.binding import RGBA, Color
    from workloads import build_scene

    print(f"card: {card()}", flush=True)
    api = forma_b200.load()
    if args.pdl is not None:
        api.set_option("pdl", args.pdl)
    comp, w, h = build_scene(api, args.workload)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    renderer = api.Renderer(0)
    renderer.set_stream(stream.cuda_stream)
    fb = torch.zeros((h, w * 4), dtype=torch.uint8, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)  # L2 flushed between frames, as bench.py does
    clear = Color(1.0, 1.0, 1.0, 0.0)

    def frame():
        renderer.render_device(comp, fb.data_ptr(), w, h, RGBA, clear, None, None, w * 4, timings=False)

    for _ in range(3):
        frame()
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(args.frames):
                with torch.cuda.stream(stream):
                    flush.zero_()
                torch.cuda.synchronize()
                with record_function("forma_frame"):
                    frame()
                torch.cuda.synchronize()
        prof.export_chrome_trace(path)
        if args.trace:
            with open(path) as f, open(args.trace, "w") as g:
                g.write(f.read())
        ops = frame_ops(path, "forma_frame")
    st = renderer.stage_times()
    print(f"workload {args.workload} {w}x{h}, last of {args.frames} frames, counters {renderer.counters()}")
    idle, boundaries = report(ops)
    print(f"stage_ms (profiled frame): " + ", ".join(f"{k} {v:.3f}" for k, v in st.items()))
    print(f"idle inside the event window: {idle:.1f} us over {len(boundaries)} boundaries")
    if not args.no_probe:
        res = run_probe()
        names = {0: "plain launches", 1: "programmatic serialization", 2: "programmatic serialization + event record between"}
        for m in (0, 1, 2):
            print(f"probe {names[m]}: us per kernel " + ", ".join(f"{v:.2f}" for v in res[m]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
