"""What the dense spike stream's store pattern costs on this GPU, next to the write ceiling and the real step kernel.

(a) A microbenchmark in the shape of the c2 step: 65 536 agents x 1 024 cells, 132-ish CTAs of 16 warps in two groups of 8,
    tiles of 32 agents.  Every warp writes its 512-B piece of each agent's rate row (st.global.cs.v4, 268 MB per pass) and,
    per pattern, the 8.4 MB spike region:
      split : as the pair loop stores it, 16 B per warp and agent from an elected lane, so each 32-B sector of a spike row
              is completed by a second warp at another time (st.global.cs);
      lines : the same bytes after the tile's rate rows, as whole 128-B lines (512 B per warp instruction);
      none  : no spike region.
    The three are timed alternately (three rounds) with torch.cuda events; the plain fill ceiling comes from bw_probe.py.
(b) The real kernel through bench.measure: c2 with and without spikes, c2e and c3, alternated three times.

    python scripts/spike_write_probe.py [--out DIR] [--steps N]

Prints one JSON object (also written to DIR/spike_write_probe.json).  Compiles the microbenchmark with nvcc into DIR.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_AGENTS, N_CELLS, TA = 65536, 1024, 32
PATTERNS = ("split", "lines", "none")

KERNEL = r"""
#include <cstdint>
#include <cuda_runtime.h>
constexpr int TA = 32, WARPS = 16, GROUP = 8;
__device__ __forceinline__ void st_cs_v4(uint32_t* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
// PATTERN 0: split 16-B spike pieces, 1: whole spike lines per tile, 2: no spike region.  Warp wg of a group owns cells
// [128 wg, 128 wg + 128) of every agent (n_cells = 128 * GROUP), like the lean consumer groups of k_step.
template <int PATTERN>
__global__ void __launch_bounds__(WARPS * 32, 1) k_probe(uint32_t* rates, uint32_t* spikes, int n_agents, uint32_t seed) {
  constexpr int n_cells = 128 * GROUP, spike_ld = n_cells / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, grp = warp / GROUP, wg = warp % GROUP;
  const int groups = gridDim.x * (WARPS / GROUP), n_tiles = n_agents / TA;
  for (int tile = blockIdx.x * (WARPS / GROUP) + grp; tile < n_tiles; tile += groups) {
    for (int a = tile * TA; a < tile * TA + TA; ++a) {
      const uint32_t h = ((uint32_t)a * 0x9E3779B9u) ^ seed ^ ((uint32_t)threadIdx.x * 0x85EBCA6Bu);
      st_cs_v4(rates + (long long)a * n_cells + 128 * wg + 4 * lane, h, h + 1u, h + 2u, h + 3u);
      if (PATTERN == 0) {
        const uint32_t b = __ballot_sync(0xffffffffu, h & 1u);
        if (lane == 0) st_cs_v4(spikes + (long long)a * spike_ld + 4 * wg, b, b ^ 1u, b ^ 2u, b ^ 3u);
      }
    }
    if (PATTERN == 1) {
      // the tile's TA rows are TA * spike_ld contiguous words: warp wg writes rows [TA/GROUP wg, TA/GROUP (wg + 1))
      uint32_t* base = spikes + ((long long)tile * TA + (TA / GROUP) * wg) * spike_ld;
      for (int w = 4 * lane; w < (TA / GROUP) * spike_ld; w += 128) {
        const uint32_t b = ((uint32_t)(tile * 4096 + wg * 512 + w) * 0x9E3779B9u) ^ seed;
        st_cs_v4(base + w, b, b ^ 1u, b ^ 2u, b ^ 3u);
      }
    }
  }
}
extern "C" int probe_launch(int pattern, void* rates, void* spikes, int n_agents, unsigned seed, void* stream) {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaStream_t s = (cudaStream_t)stream;
  if (pattern == 0) k_probe<0><<<sms, WARPS * 32, 0, s>>>((uint32_t*)rates, (uint32_t*)spikes, n_agents, seed);
  else if (pattern == 1) k_probe<1><<<sms, WARPS * 32, 0, s>>>((uint32_t*)rates, (uint32_t*)spikes, n_agents, seed);
  else k_probe<2><<<sms, WARPS * 32, 0, s>>>((uint32_t*)rates, (uint32_t*)spikes, n_agents, seed);
  return (int)cudaGetLastError();
}
"""


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:           # (the numbers still stand; say where the card's identity is missing)
        return {"error": repr(e)}


def build_probe(out_dir):
    src = os.path.join(out_dir, "spike_write_probe.cu")
    lib = os.path.join(out_dir, "spike_write_probe.so")
    with open(src, "w") as f:
        f.write(KERNEL)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                    "-shared", src, "-o", lib], check=True)
    return lib


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "all": xs}


def micro(torch, lib_path, launches=20, rounds=3):
    lib = ctypes.CDLL(lib_path)
    lib.probe_launch.restype = ctypes.c_int
    lib.probe_launch.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_uint, ctypes.c_void_p]
    rates = torch.empty(N_AGENTS * N_CELLS, dtype=torch.int32, device="cuda")
    spikes = torch.empty(N_AGENTS * N_CELLS // 32, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def run(p, n, seed):
        for i in range(n):
            rc = lib.probe_launch(p, rates.data_ptr(), spikes.data_ptr(), N_AGENTS, seed + i, stream)
            assert rc == 0, f"probe launch failed ({rc})"

    for p in range(len(PATTERNS)):
        run(p, 5, 1)
    torch.cuda.synchronize()
    us = {k: [] for k in PATTERNS}
    for r in range(rounds):
        for p, name in enumerate(PATTERNS):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(p, launches, 100 * r)
            e1.record()
            torch.cuda.synchronize()
            us[name].append(e0.elapsed_time(e1) * 1e3 / launches)
    rate_bytes, spike_bytes = N_AGENTS * N_CELLS * 4, N_AGENTS * N_CELLS // 8
    res = {}
    for name in PATTERNS:
        b = rate_bytes + (0 if name == "none" else spike_bytes)
        res[name] = {"us": spread(us[name]), "bytes": b, "gbs_median": b / (statistics.median(us[name]) * 1e-6) / 1e9}
    res["split_minus_lines_us"] = statistics.median(us["split"]) - statistics.median(us["lines"])
    res["split_slower_outside_spread"] = min(us["split"]) > max(us["lines"])
    del rates, spikes
    torch.cuda.empty_cache()
    return res


def fill_ceiling():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "bw_probe.py")], capture_output=True, text=True, check=True)
    return json.loads(out.stdout.strip().splitlines()[-1])


def real_kernel(torch, steps, rounds=3):
    import bench
    import ratinabox_b200 as rb
    from ratinabox_b200 import _lib
    lib = _lib.load()
    cases = [("c2", True), ("c2", False), ("c2e", True), ("c3", True)]
    got = {f"{n}{'' if s else '_no_spikes'}": [] for n, s in cases}
    for _ in range(rounds):
        for name, spikes in cases:
            r = bench.measure(rb, lib, torch, None, name, steps, 20, 0, 1, 0, spikes=spikes, e2e=False)
            got[f"{name}{'' if spikes else '_no_spikes'}"].append(r["ms_per_step"] * 1e3)
    return {k: {"us_per_step": spread(v)} for k, v in got.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for the compiled probe and the JSON (default: a temporary one)")
    ap.add_argument("--steps", type=int, default=300, help="timed steps per bench.measure call")
    args = ap.parse_args()
    out_dir = args.out or tempfile.mkdtemp(prefix="spike_write_probe_")
    os.makedirs(out_dir, exist_ok=True)
    import torch
    assert torch.cuda.is_available(), "spike_write_probe needs a GPU"
    lib_path = build_probe(out_dir)
    res = {"gpu": gpu_info(), "shape": f"{N_AGENTS} agents x {N_CELLS} cells, tiles of {TA} agents"}
    res["micro"] = micro(torch, lib_path)
    res["fill_ceiling"] = fill_ceiling()
    res["real"] = real_kernel(torch, args.steps)
    res["gpu_after"] = gpu_info()
    line = json.dumps(res)
    with open(os.path.join(out_dir, "spike_write_probe.json"), "w") as f:
        f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
