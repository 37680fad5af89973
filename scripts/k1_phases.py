"""Where K1 (the FAST extraction kernel of the k21 benchmark) spends a window, phase by phase, on the GPU.

    python scripts/k1_phases.py [--lib PATH] [--bases N] [--size S] [--steps K] [--out DIR]

Builds (or takes with --lib) a copy of libjfgpu.so compiled with -DJF_K1_PROF=1, in which the FAST extract_kernel
instantiations stamp clock64() around each of their block barriers (jf_extract.cuh, `bsync`); the product build compiles
without the stamps, so no kernel of it changes.  Counts the benchmark's k21 workload (synthetic FASTA resident in HBM,
-s 8G, canonical) like bench.py's `value` arm and prints one JSON line: per segment of a window -- each ended by a block
barrier -- the mean cycles a warp spends working in it and waiting at its barrier, the hashing part of the E appends,
the whole window, and K1's time per step in this build (the stamps and their extra spills make it a little slower than
the product kernel).  The build goes to a temporary directory; nothing is written in the tree.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEGS = ["tma_wait", "B_classify", "C_scan", "C_stream_or", "D_pre", "E_append", "ring_pass", "E_end", "window_end"]
WORDS = 2 * len(SEGS) + 4


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return q.splitlines()[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def build_lib(tmp):
    out = os.path.join(tmp, "lib")
    csrc = os.path.join(ROOT, "jellyfish_b200", "csrc")
    subprocess.check_call(["make", "-C", csrc, "OUT=" + out, "NVEXTRA=-DJF_K1_PROF=1", os.path.join(out, "libjfgpu.so")],
                          stdout=subprocess.DEVNULL)
    return os.path.join(out, "libjfgpu.so")


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default=None, help="a libjfgpu.so built with NVEXTRA=-DJF_K1_PROF=1 (default: build one)")
    ap.add_argument("--bases", type=int, default=5_000_000_000)
    ap.add_argument("--size", default="8G")
    ap.add_argument("--k", type=int, default=21)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()

    with tempfile.TemporaryDirectory() as tmp:
        lib_path = a.lib or build_lib(tmp)
        from jellyfish_b200 import _lib
        _lib.LIB_PATH = lib_path
        lib = _lib.load()
        if not hasattr(lib, "jfgpu_k1_prof"):
            raise SystemExit("%s was not built with -DJF_K1_PROF=1" % lib_path)
        lib.jfgpu_k1_prof.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
        lib.jfgpu_k1_prof.restype = C.c_int
        import torch
        from jellyfish_b200 import HashCounter
        import bench

        dev = torch.device("cuda", 0)
        nbytes = lib.jfgpu_synth_fasta_bytes(a.bases)
        text = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
        got = C.c_uint64(0)
        rc = lib.jfgpu_synth_fasta_device(0, C.c_void_p(text.data_ptr()), nbytes + 256, a.bases, 0x9E3779B97F4A7C15, C.byref(got), None)
        assert rc == 0, "synthetic FASTA generation failed"
        torch.cuda.synchronize()
        acc = (C.c_ulonglong * WORDS)()
        hc = HashCounter(bench.parse_size(a.size), 7, k=a.k, canonical=True, device=0)

        def step():
            hc.clear()
            hc.add_device_text(text.data_ptr(), got.value)
            return hc.done()

        for _ in range(a.warmup):
            step()
        assert lib.jfgpu_k1_prof(acc, WORDS) == 0
        k1_s = 0.0
        for _ in range(a.steps):
            st = step()
            k1_s += st["seconds_count_kernel"]
        assert lib.jfgpu_k1_prof(acc, WORDS) == 0
        hc.close()
        v = list(acc)
        windows, ctas = v[2 * len(SEGS) + 2], v[2 * len(SEGS) + 3]
        assert windows > 0, "the FAST kernel did not run (no phase counters)"
        warp_windows = 32.0 * windows          # NTH = 1024: 32 warps per CTA
        seg = {}
        for i, name in enumerate(SEGS):
            work, wait = v[2 * i] / warp_windows, v[2 * i + 1] / warp_windows
            seg[name] = {"cycles": round(work + wait, 1), "work": round(work, 1), "barrier_wait": round(wait, 1)}
        loop = v[2 * len(SEGS) + 1] / warp_windows
        print(json.dumps({
            "bench": "k1_phases", "k": a.k, "bases": a.bases, "size": a.size, "steps": a.steps, "gpu": gpu_info(),
            "windows_per_step": windows // a.steps, "ctas_per_step": ctas // a.steps,
            "k1_ms_per_step_instrumented": round(1e3 * k1_s / a.steps, 2),
            "cycles_per_window": round(loop, 1),
            "segments_per_window": seg,
            "E_hash_cycles_per_warp_window": round(v[2 * len(SEGS)] / warp_windows, 1),
            "barriers_per_window": 13,
            "note": "cycles = SM clock cycles (clock64) per window, averaged over warps; a segment ends at a block barrier; "
                    "E_append and ring_pass are summed over the 4 ring passes of a window",
        }))


if __name__ == "__main__":
    main()
