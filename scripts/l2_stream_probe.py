"""How fast can every SM stream one L2-resident weight image into shared memory? (developer tool, needs an H100)

The trunk kernel streams its 256 KB fp16 W3 image through a shared-memory ring once per tile, on every SM at once.
This probe builds a tiny kernel in a temporary directory that does only that: one CTA per SM, a producer thread
bulk-copies (cp.async.bulk) the same 256 KB image into a ring of 16 KB slots, completion counted on mbarriers, and a
consumer warp hands every slot back as soon as it has landed.  It reports the aggregate rate into shared memory, with
the card's name and power limit, for several ring depths.

    python scripts/l2_stream_probe.py [--reps 400]
"""
import _harness
import argparse
import os
import subprocess
import tempfile

SRC = r"""
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr uint32_t SLOT = 16384, IMG = 16 * SLOT;

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile("{\n\t.reg .pred p;\n\tW:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@!p bra W;\n\t}"
               ::"r"(bar), "r"(parity) : "memory");
}

__global__ void __launch_bounds__(64, 1) stream_kernel(const unsigned char *img, int reps, int nslot, unsigned *sink) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ unsigned long long full[16], empty[16];
  const uint32_t ring = (uint32_t)__cvta_generic_to_shared(smem);
  const uint32_t full_s = (uint32_t)__cvta_generic_to_shared(full), empty_s = (uint32_t)__cvta_generic_to_shared(empty);
  if (threadIdx.x == 0) {
    for (int i = 0; i < nslot; i++) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(full_s + 8 * i));
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(empty_s + 8 * i));
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int total = reps * (int)(IMG / SLOT);
  if (threadIdx.x == 0) {            // producer
    for (int gs = 0; gs < total; gs++) {
      const int s = gs % nslot;
      mbar_wait(empty_s + 8 * s, ((gs / nslot) & 1) ^ 1);
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full_s + 8 * s), "r"(SLOT) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"(ring + s * SLOT), "l"(img + (size_t)(gs % (IMG / SLOT)) * SLOT), "r"(SLOT), "r"(full_s + 8 * s)
                   : "memory");
    }
  } else if (threadIdx.x == 32) {    // consumer: touch one word of every slot, hand it back
    unsigned acc = 0;
    for (int gs = 0; gs < total; gs++) {
      const int s = gs % nslot;
      mbar_wait(full_s + 8 * s, (gs / nslot) & 1);
      acc += *reinterpret_cast<volatile unsigned *>(smem + s * SLOT + (gs & 63) * 4);
      asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(empty_s + 8 * s) : "memory");
    }
    if (acc == 0x12345678u) *sink = acc;
  }
}

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

int main(int argc, char **argv) {
  const int reps = argc > 1 ? atoi(argv[1]) : 400;
  int dev = 0, sms = 0;
  CK(cudaSetDevice(dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  unsigned char *img; unsigned *sink;
  CK(cudaMalloc(&img, IMG)); CK(cudaMalloc(&sink, 4));
  CK(cudaMemset(img, 1, IMG));
  CK(cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 12 * SLOT));
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  const int depths[] = {2, 4, 6, 8, 12};
  for (int nslot : depths) {
    stream_kernel<<<sms, 64, nslot * SLOT>>>(img, 20, nslot, sink);   // warm-up: image into L2, module loaded
    CK(cudaGetLastError());
    float best = 1e30f;
    for (int r = 0; r < 5; r++) {
      CK(cudaEventRecord(a));
      stream_kernel<<<sms, 64, nslot * SLOT>>>(img, reps, nslot, sink);
      CK(cudaEventRecord(b));
      CK(cudaEventSynchronize(b));
      float ms; CK(cudaEventElapsedTime(&ms, a, b));
      if (ms < best) best = ms;
    }
    const double bytes = (double)sms * reps * IMG;
    printf("ring %2d x 16 KB: %d CTAs x %d passes of 256 KB in %.3f ms -> %.2f TB/s into shared memory\n", nslot,
           sms, reps, best, bytes / best / 1e9);
  }
  return 0;
}
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=400, help="passes over the 256 KB image per CTA")
    args = ap.parse_args()
    print("card:", _harness.card())
    with tempfile.TemporaryDirectory(prefix="cg_l2probe_") as td:
        src, exe = os.path.join(td, "probe.cu"), os.path.join(td, "probe")
        with open(src, "w") as f:
            f.write(SRC)
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-o", exe, src])
        out = subprocess.run([exe, str(args.reps)], capture_output=True, text=True)
        print(out.stdout, end="")
        print(f"SM clock after the run: {_harness.smi('clocks.sm')}")
        if out.returncode != 0:
            raise SystemExit(out.returncode)


if __name__ == "__main__":
    main()
