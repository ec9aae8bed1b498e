"""Developer probe (not the bench contract): how fast can the headline mat-vec's ring stream at all?

Compiles (nvcc, into a temporary directory) a kernel with the headline's exact TMA ring -- 132 x `resident` CTAs, a producer warp issuing
cp.async.bulk into `stages` stages of `rows` x 2304 bytes, chunks after the first handed out by an atomic counter, programmatic dependent
launch between consecutive launches -- whose consumer warps wait on each full barrier and release the stage without computing anything.
It times that kernel over the bench sweep (13 distinct Q4_K 4096 x 11008 matrices, 330 MB) in a CUDA graph with device events, and in
the same process the real sweep through ggml_b200.mul_mat with SRC0_STATIC | SRC1_STATIC, alternating the two.  The gap between the two
rates bounds what any change to the consume phase can gain at the card's power limit.

Usage: python scripts/sb_stream_ceiling.py [--rounds 3] [--seconds 1.5] [--json OUT]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402  (sweep definition, weight generator, clock sampler)

K, M, TYPE = 4096, 11008, 12
ROW_BYTES = K // 256 * 144

PROBE_CU = r"""
#include "b200_ptx.cuh"
#include <cuda_runtime.h>
using namespace b200;

constexpr int MAX_STAGES = 6, CONSUMER_WARPS = 4;

// the superblock mat-vec's ring with an empty consume phase
__global__ void __launch_bounds__((CONSUMER_WARPS + 1) * 32, 4)
sb_ring_probe(const uint8_t * w, int64_t M, int row_bytes, int rows_per_chunk, int nchunks, int stage_bytes, int nstages, unsigned * counters) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t * stages = smem;
    uint64_t * full = (uint64_t *)(stages + (size_t)nstages * stage_bytes);
    uint64_t * empty = full + MAX_STAGES;
    int * chunk_of = (int *)(empty + MAX_STAGES);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pdl_launch_dependents();
    if (tid == 0) {
        for (int s = 0; s < nstages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], CONSUMER_WARPS); }
        mbar_fence_init();
    }
    __syncthreads();
    auto issue = [&](int s, int chunk) {
        chunk_of[s] = chunk < nchunks ? chunk : -1;
        if (chunk < nchunks) {
            const int64_t row0 = (int64_t)chunk * rows_per_chunk;
            const uint32_t bytes = (uint32_t)min((int64_t)rows_per_chunk, M - row0) * (uint32_t)row_bytes;
            mbar_expect_tx(&full[s], bytes);
            bulk_g2s(stages + (size_t)s * stage_bytes, w + (size_t)row0 * row_bytes, bytes, &full[s]);
        } else {
            mbar_arrive(&full[s]);
        }
    };
    if (warp == CONSUMER_WARPS) {
        if (lane == 0) {
            issue(0, (int)blockIdx.x);
            int it = 1;
            bool done = (int)blockIdx.x >= nchunks;
            while (!done) {
                const int s = it % nstages;
                const int chunk = (int)atomicAdd(&counters[0], 1u) + (int)gridDim.x;
                if (it >= nstages) mbar_wait(&empty[s], (uint32_t)((it / nstages) - 1) & 1u);
                issue(s, chunk);
                done = chunk >= nchunks;
                ++it;
            }
            __threadfence();
            if (atomicAdd(&counters[1], 1u) == gridDim.x - 1) { counters[0] = 0; counters[1] = 0; __threadfence(); }
        }
        return;
    }
    for (int it = 0;; ++it) {
        const int s = it % nstages;
        mbar_wait(&full[s], (uint32_t)(it / nstages) & 1u);
        if (chunk_of[s] < 0) break;
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }
    if (tid == 0) pdl_wait();                 // completion stays transitive along the stream, as in the mat-vec kernel
}

extern "C" int sb_ring_probe_launch(const void * w, long long M, int row_bytes, int rows_per_chunk, int stage_bytes, int nstages, int grid,
                                    unsigned * counters, void * stream) {
    const int nchunks = (int)((M + rows_per_chunk - 1) / rows_per_chunk);
    const int smem = nstages * stage_bytes + 2 * MAX_STAGES * 8 + MAX_STAGES * 4 + 64;
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(sb_ring_probe, cudaFuncAttributeMaxDynamicSharedMemorySize, 222 * 1024) != cudaSuccess) return 1;
        attr = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid < nchunks ? grid : nchunks); cfg.blockDim = dim3((CONSUMER_WARPS + 1) * 32);
    cfg.dynamicSmemBytes = smem; cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, sb_ring_probe, (const uint8_t *)w, (int64_t)M, row_bytes, rows_per_chunk, nchunks, stage_bytes, nstages, counters) == cudaSuccess ? 0 : 2;
}
"""


def build_probe(tmp: Path) -> C.CDLL:
    src = tmp / "sb_ring_probe.cu"
    so = tmp / "libsb_ring_probe.so"
    src.write_text(PROBE_CU)
    nvcc = os.environ.get("NVCC") or ("/usr/local/cuda/bin/nvcc" if Path("/usr/local/cuda/bin/nvcc").exists() else "nvcc")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
                    f"-I{ROOT / 'ggml_b200' / 'csrc'}", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    L.sb_ring_probe_launch.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.sb_ring_probe_launch.restype = C.c_int
    return L


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, mx = (f.strip() for f in out.split(","))
        return {"name": name, "power_limit": plim, "sm_max_clock": mx}
    except Exception as e:
        return {"name": None, "error": str(e)[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternating probe / real windows")
    ap.add_argument("--seconds", type=float, default=1.5, help="device time per window")
    ap.add_argument("--resident", type=int, default=4)
    ap.add_argument("--stages", type=int, default=2)
    ap.add_argument("--rows", type=int, default=8, help="rows per chunk (stage = rows x 2304 B)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nbuf = bench.NBUF
    Ws = bench.make_weights(torch, TYPE, nbuf, K, M, seed=1234)
    X = torch.rand(K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5678)) * 2 - 1
    Ys = [torch.empty((1, 1, 1, M), dtype=torch.float32, device="cuda") for _ in range(nbuf)]
    F_IND = g.MM_SRC0_STATIC | g.MM_SRC1_STATIC
    wb = ROW_BYTES * M
    stage_bytes = (args.rows * ROW_BYTES + 127) & ~127
    counters = torch.zeros(64 * 8, dtype=torch.int32, device="cuda")
    slot = [0]

    with tempfile.TemporaryDirectory(prefix="sb_ring_probe_") as tmp:
        P = build_probe(Path(tmp))

        def probe_sweep():
            st = torch.cuda.current_stream().cuda_stream
            for i in range(nbuf):
                ctr = counters.data_ptr() + (slot[0] % 64) * 8 * 4
                slot[0] += 1
                rc = P.sb_ring_probe_launch(Ws[i].data_ptr(), M, ROW_BYTES, args.rows, stage_bytes, args.stages, sms * args.resident, ctr, st)
                assert rc == 0, f"probe launch failed ({rc})"

        def real_sweep():
            for i in range(nbuf):
                g.mul_mat(TYPE, Ws[i], X, M, 1, K, out=Ys[i], flags=F_IND)

        graphs = {}
        for name, fn in (("probe", probe_sweep), ("real", real_sweep)):
            fn(); torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                for _ in range(bench.SWEEPS_PER_GRAPH):
                    fn()
            graphs[name] = gr

        def window(name):
            gr = graphs[name]
            for _ in range(3):
                gr.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); gr.replay(); e1.record(); torch.cuda.synchronize()
            reps = max(5, int(args.seconds / max(e0.elapsed_time(e1) * 1e-3, 1e-6)))
            sampler = bench.ClockSampler(0)
            sampler.start()
            t0 = sampler.mark()
            e0.record()
            for _ in range(reps):
                gr.replay()
            e1.record()
            torch.cuda.synchronize()
            t1 = sampler.mark()
            clocks = sampler.stop(t0, t1)
            n = reps * bench.SWEEPS_PER_GRAPH * nbuf
            us = e0.elapsed_time(e1) * 1e3 / n
            return {"GBps": wb / us / 1e3, "us_per_matvec": us, "matvecs": n, "sm_mhz": clocks.get("sm_mhz"), "power_w_max": clocks.get("power_w_max"),
                    "reasons": clocks.get("reasons")}

        rounds = []
        for _ in range(args.rounds):
            rounds.append({"probe": window("probe"), "real": window("real")})

    probe = statistics.median(r["probe"]["GBps"] for r in rounds)
    real = statistics.median(r["real"]["GBps"] for r in rounds)
    res = {"card": card(), "shape": f"q4_K {K}x{M} n=1, {nbuf} distinct matrices ({nbuf * wb / 1e6:.0f} MB) per sweep",
           "ring": {"ctas": sms * args.resident, "stages": args.stages, "stage_bytes": stage_bytes, "rows_per_chunk": args.rows},
           "act_regs_env": os.environ.get("GGML_B200_SB_ACT_REGS"),
           "probe_GBps_median": probe, "real_GBps_median": real, "real_over_probe": real / probe, "rounds": rounds}
    print(json.dumps(res), flush=True)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
