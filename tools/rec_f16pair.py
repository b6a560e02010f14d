"""Tensor-core rates behind the fp16-pair GRU-256 recurrence (rec_fwd_h16_kernel) and the per-launch recurrence time.

1. Microbenchmark: dependent-chain latency and per-SM throughput of warp-level mma.sync m16n8k16 f16 -> f32 (HMMA.16816.F32)
   against m16n8k8 tf32 (HMMA.1688.F32.TF32), measured with clock64 in a small CUDA program compiled into a temporary
   directory (nvcc, sm_90a).
2. With --rec: the recurrence launches of the no-grad fused forward (GRU 256 -> 256, 2 layers, LayerNorm prologue,
   time sum, B = 128, T = 120, as in the fuse step) timed with torch.profiler; run it once per build
   (B200RNN_LIB=<other build>/libb200rnn.so) to compare builds.

Prints one JSON line. Needs an H100.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <cstdio>
#include <cstdint>
__device__ __forceinline__ void mma16(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void mma8(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// CHAINS independent accumulators per warp, ITERS rounds; per warp: cycles of the loop
template <int K16, int CHAINS>
__global__ void bench(int iters, long long* cycles, float* sink, uint32_t seed) {
  uint32_t a[4], b[2];
  for (int i = 0; i < 4; ++i) a[i] = seed * (threadIdx.x + i + 1) & 0x3bff3bffu;
  for (int i = 0; i < 2; ++i) b[i] = seed * (threadIdx.x + 7 * i + 3) & 0x3bff3bffu;
  float d[CHAINS][4] = {};
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it)
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) { if (K16) mma16(d[c], a, b); else mma8(d[c], a, b); }
  const long long t1 = clock64();
  float s = 0.f;
  for (int c = 0; c < CHAINS; ++c) s += d[c][0] + d[c][1] + d[c][2] + d[c][3];
  sink[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x % 32 == 0) cycles[blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32] = t1 - t0;
}
template <int K16, int CHAINS>
double run(int blocks, int warps, int iters, double* mma_per_clk_sm) {
  long long* cyc; float* sink;
  cudaMalloc(&cyc, sizeof(long long) * blocks * warps);
  cudaMalloc(&sink, sizeof(float) * blocks * warps * 32);
  bench<K16, CHAINS><<<blocks, warps * 32>>>(iters, cyc, sink, 12345u);  // warm-up
  bench<K16, CHAINS><<<blocks, warps * 32>>>(iters, cyc, sink, 12345u);
  cudaDeviceSynchronize();
  long long* h = new long long[blocks * warps];
  cudaMemcpy(h, cyc, sizeof(long long) * blocks * warps, cudaMemcpyDeviceToHost);
  double mx = 0;
  for (int i = 0; i < blocks * warps; ++i) mx = h[i] > mx ? h[i] : mx;
  delete[] h;
  cudaFree(cyc); cudaFree(sink);
  // one block per SM: MMAs the SM issued over the slowest warp's cycles
  *mma_per_clk_sm = (double)warps * CHAINS * iters / mx;
  return mx / ((double)CHAINS * iters);  // cycles per MMA of one warp
}
int main() {
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  double t;
  const double lat16 = run<1, 1>(1, 1, 4096, &t), lat8 = run<0, 1>(1, 1, 4096, &t);
  double thr16, thr8;
  run<1, 8>(sms, 16, 2048, &thr16);
  run<0, 8>(sms, 16, 2048, &thr8);
  printf("{\"latency_cycles\": {\"m16n8k16_f16\": %.2f, \"m16n8k8_tf32\": %.2f}, "
         "\"mma_per_cycle_per_sm\": {\"m16n8k16_f16\": %.3f, \"m16n8k8_tf32\": %.3f}, "
         "\"macs_per_cycle_per_sm\": {\"m16n8k16_f16\": %.0f, \"m16n8k8_tf32\": %.0f}}\n",
         lat16, lat8, thr16, thr8, thr16 * 16 * 8 * 16, thr8 * 16 * 8 * 8);
  return cudaGetLastError() != cudaSuccess;
}
"""


def microbench():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "mma.cu"), os.path.join(d, "mma")
        with open(src, "w") as f:
            f.write(SRC)
        subprocess.run(["nvcc", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", src, "-o", exe], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    return json.loads(out)


def rec_times(steps):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "icassp2022-depression_b200")]
    import torch
    from torch.profiler import ProfilerActivity, profile

    import b200rnn

    torch.manual_seed(0)
    gru = b200rnn.GRU(256, 256, num_layers=2, batch_first=True).to("cuda:0")
    ln = torch.nn.LayerNorm(256).to("cuda:0")
    x = torch.randn(128, 120, 256, device="cuda:0")
    with torch.no_grad():
        for _ in range(10):
            gru.forward_ln_sum(x, ln)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(steps):
            gru.forward_ln_sum(x, ln)
        ev[1].record()
        torch.cuda.synchronize()
        call_ms = ev[0].elapsed_time(ev[1]) / steps
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                gru.forward_ln_sum(x, ln)
            torch.cuda.synchronize()
    rec = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "rec_fwd" in e.name:
            name = e.name.split("rec_fwd_")[1].split("<")[0].split("I")[0]
            rec.setdefault(name, []).append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
    launches = {k: {"n": len(v), "mean_us": sum(v) / len(v)} for k, v in rec.items()}
    return {"lib": b200rnn._lib.LIB_PATH, "call_ms": call_ms, "rec_launches": launches}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rec", action="store_true", help="time the recurrence launches of the fused forward")
    ap.add_argument("--no-mma", action="store_true", help="skip the mma.sync microbenchmark")
    ap.add_argument("--steps", type=int, default=50)
    a = ap.parse_args()
    out = {}
    if not a.no_mma:
        out["mma"] = microbench()
    if a.rec:
        out["rec"] = rec_times(a.steps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
