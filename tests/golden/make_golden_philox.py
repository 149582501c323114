"""Writes tests/golden/philox4x32_10.json: known answers of Philox4x32-10 from the CUDA toolkit's own
curand_Philox4x32_10 (curand_philox4x32_x.h), compiled as host code with nvcc. The sampler kernel calls the same
function; tests/sampling_refs.py restates it in numpy and tests/test_sampling_host.py checks that restatement here.

    python tests/golden/make_golden_philox.py        (needs nvcc; no GPU)
"""
import json
import os
import shutil
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "philox4x32_10.json")

M = 0xFFFFFFFF
# (counter c0..c3, key k0, k1): all zeros, all ones, and mixed values including the counters the sampler uses
VECTORS = [
    ((0, 0, 0, 0), (0, 0)),
    ((M, M, M, M), (M, M)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0)),
    ((1, 2, 3, 4), (5, 6)),
    ((0, 0, 0, 0), (M, M)),
    ((M, M, M, M), (0, 0)),
    ((7, 255, 1021, 0), (12345, 0)),
    ((31, 65536, 65534, 5), (0xDEADBEEF, 0xCAFEF00D)),
    ((0x80000000, 1, 0, 1), (1, 0x80000000)),
]

SRC = r"""
#include <cstdio>
#include <cuda_runtime.h>
#define QUALIFIERS static inline __host__ __device__
#include <curand_philox4x32_x.h>
int main() {
  unsigned v[6];
  while (scanf("%u %u %u %u %u %u", &v[0], &v[1], &v[2], &v[3], &v[4], &v[5]) == 6) {
    uint4 r = curand_Philox4x32_10(make_uint4(v[0], v[1], v[2], v[3]), make_uint2(v[4], v[5]));
    printf("%u %u %u %u\n", r.x, r.y, r.z, r.w);
  }
  return 0;
}
"""


def main():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, "philox.cu"), os.path.join(tmp, "philox")
        with open(src, "w") as f:
            f.write(SRC)
        subprocess.run([nvcc, "-Wno-deprecated-gpu-targets", "-o", exe, src], check=True)
        inp = "".join(" ".join(str(x) for x in c + k) + "\n" for c, k in VECTORS)
        res = subprocess.run([exe], input=inp, capture_output=True, text=True, check=True).stdout.split("\n")
    cases = [{"counter": list(c), "key": list(k), "out": [int(x) for x in line.split()]}
             for (c, k), line in zip(VECTORS, res)]
    with open(OUT, "w") as f:
        json.dump({"generator": "curand_Philox4x32_10, CUDA toolkit host build", "cases": cases}, f, indent=1)
    print(f"wrote {OUT}: {len(cases)} vectors")


if __name__ == "__main__":
    main()
