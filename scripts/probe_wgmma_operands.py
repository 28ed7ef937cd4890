"""Clocks per m64n32k16 bf16 wgmma with the A operand in shared memory or in registers (H100, sm_90a).

The whole-attempt linear kernel (torchdiffeq_b200/csrc/tdq_attempt.cu) issues 48 m64n32k16 products per warpgroup and
tile-stage, from two warpgroups per SM.  An A operand in shared memory adds 2 KB of shared-memory traffic to the 1 KB of
its B operand; this probe measures what that costs.  One CTA of two warpgroups per SM issues rounds of 48 products, in
three forms:
  smem   every A operand from shared memory (the stage kernels' form)
  regs   every A operand from registers
  mixed  40 register-A and 8 shared-A products per 48 (the attempt kernel with the hi and mid weight planes in registers)
and reports SM clocks per product (both warpgroups' products counted: the tensor pipe and shared memory are per SM).

    python scripts/probe_wgmma_operands.py [--rounds N]

Compiles a small CUDA program with nvcc into a temporary directory and prints one JSON line.  Needs a GPU.
"""
import argparse
import json
import os
import shutil
import subprocess
import tempfile

SRC = r"""
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint64_t desc(uint32_t a) {   // no swizzle, LBO 128, SBO 2048
    return (uint64_t)((a & 0x3FFFFu) >> 4) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(2048 >> 4) << 32);
}
#define ACC16 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
__device__ __forceinline__ void mma_ss(float (&d)[16], uint64_t da, uint64_t db) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, 1, 1, 1, 0, 1;\n"
                 : ACC16 : "l"(da), "l"(db));
}
__device__ __forceinline__ void mma_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t db) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, 1, 1, 1, 1;\n"
                 : ACC16 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

// NS of every 48 products read A from shared memory (the last NS of each round), the others from registers
template <int NS>
__global__ void __launch_bounds__(256, 1) k_probe(int rounds, float *out, long long *clk) {
    extern __shared__ __align__(128) uint8_t sm[];
    const int tid = threadIdx.x, h = tid >> 7;
    for (int i = tid; i < 3 * 32768 / 4 + 2 * 8192 / 4; i += 256)          // small bf16 pairs, not all zero
        reinterpret_cast<uint32_t *>(sm)[i] = 0x3c003c00u ^ ((i * 2654435761u) & 0x007f007fu);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const uint32_t base = (uint32_t)__cvta_generic_to_shared(sm);
    const uint32_t wa = base + h * 16384, wb = base + 3 * 32768 + h * 8192;   // A: 3 planes of 64 x 128; B: 32 x 128
    uint32_t a[8][4];
#pragma unroll
    for (int ks = 0; ks < 8; ++ks)
#pragma unroll
        for (int r = 0; r < 4; ++r) a[ks][r] = 0x3c003c00u ^ (uint32_t)(tid * 8 + ks * 4 + r);
    float acc[3][16];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int r = 0; r < 16; ++r) acc[c][r] = 0.f;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < rounds; ++it) {
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
        for (int p = 0; p < 48; ++p) {
            const int ks = p & 7, pl = (p >> 3) % 3;
            const uint64_t db = desc(wb + ks * 256);
            if (p >= 48 - NS) mma_ss(acc[p % 3], desc(wa + pl * 32768 + ks * 256), db);
            else mma_rs(acc[p % 3], a[ks], db);
        }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    }
    __syncthreads();
    const long long t1 = clock64();
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int r = 0; r < 16; ++r) s += acc[c][r];
    out[blockIdx.x * 256 + tid] = s;
    if (tid == 0) clk[blockIdx.x] = t1 - t0;
}

template <int NS> double run(int sms, int rounds, float *out, long long *clk) {
    const int smem = 3 * 32768 + 2 * 8192 + 16 * 1024;    // 128 KB: keeps a second CTA off the SM
    cudaFuncSetAttribute(k_probe<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    k_probe<NS><<<sms, 256, smem>>>(rounds / 10, out, clk);                    // warm-up
    k_probe<NS><<<sms, 256, smem>>>(rounds, out, clk);
    if (cudaDeviceSynchronize() != cudaSuccess) { printf("{\"error\": \"%s\"}\n", cudaGetErrorString(cudaGetLastError())); return -1; }
    long long h[1024];
    cudaMemcpy(h, clk, sms * sizeof(long long), cudaMemcpyDeviceToHost);
    double m = 0;
    for (int i = 0; i < sms; ++i) m += (double)h[i];
    return m / sms / ((double)rounds * 48 * 2);                 // SM clocks per product, both warpgroups counted
}

int main(int argc, char **argv) {
    const int rounds = argc > 1 ? atoi(argv[1]) : 20000;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    float *out;
    long long *clk;
    cudaMalloc(&out, sms * 256 * sizeof(float));
    cudaMalloc(&clk, sms * sizeof(long long));
    const double ss = run<48>(sms, rounds, out, clk), rs = run<0>(sms, rounds, out, clk), mx = run<8>(sms, rounds, out, clk);
    printf("{\"sms\": %d, \"rounds\": %d, \"clk_per_product\": {\"smem\": %.3f, \"regs\": %.3f, \"mixed_40_8\": %.3f}}\n",
           sms, rounds, ss, rs, mx);
    return 0;
}
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20000)
    args = ap.parse_args()
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "probe.cu"), os.path.join(d, "probe")
        with open(src, "w") as f:
            f.write(SRC)
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-o", exe, src], check=True)
        r = subprocess.run([exe, str(args.rounds)], capture_output=True, text=True, check=True)
    line = json.loads(r.stdout.strip().splitlines()[-1])
    try:
        import torch
        line["device"] = torch.cuda.get_device_name(0)
    except Exception:  # the probe itself does not need torch
        pass
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
