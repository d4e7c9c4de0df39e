"""Writes tests/golden/curand/philox.npz: the raw curand4 words of curandStatePhilox4_32_10_t after curand_init(seed, subsequence, 0),
for the seeds, subsequences and draw blocks densification uses (the kernel keys Philox by (seed, composed parent index) and takes
five curand_normal4 per parent, each from one curand4).

curand_kernel.h is compiled for the host (QUALIFIERS made __host__ __device__), so this runs without a GPU.  Only the words are
stored: the host branch of _curand_box_muller uses sinf / cosf where the device uses __sincosf, so host-side normals are not the
device's.  oracle/densify64.py restates the words in exact integer arithmetic and is pinned to this file by
tests/test_densify64_cpu.py.

    python tests/golden/make_philox_golden.py
"""
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "curand", "philox.npz")  # not golden/*.npz: the rasterizer tests take each of those as a scene
SEEDS = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 62 - 1]
SUBSEQUENCES = [0, 1, 255, 256, 2 ** 31 - 1, 2 ** 32]
BLOCKS = 5

SRC = r"""
#include <cstdio>
#include <cstdlib>
#include <curand_kernel.h>
int main(int argc, char **argv) {
    const unsigned long long seed = strtoull(argv[1], 0, 10), sub = strtoull(argv[2], 0, 10);
    const int blocks = atoi(argv[3]);
    curandStatePhilox4_32_10_t st;
    curand_init(seed, sub, 0ULL, &st);
    for (int n = 0; n < blocks; n++) {
        const uint4 w = curand4(&st);
        printf("%u %u %u %u\n", w.x, w.y, w.z, w.w);
    }
    return 0;
}
"""


def main():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "words.cu"), os.path.join(d, "words")
        with open(src, "w") as f:
            f.write(SRC)
        subprocess.check_call([nvcc, "-O2", "-DQUALIFIERS=static __forceinline__ __host__ __device__", src, "-o", exe])
        words = np.zeros((len(SEEDS), len(SUBSEQUENCES), BLOCKS, 4), dtype=np.uint32)
        for a, s in enumerate(SEEDS):
            for b, q in enumerate(SUBSEQUENCES):
                out = subprocess.check_output([exe, str(s), str(q), str(BLOCKS)], text=True).split()
                words[a, b] = np.array([int(v) for v in out], dtype=np.uint64).reshape(BLOCKS, 4)
    np.savez_compressed(OUT, seeds=np.array(SEEDS, dtype=np.uint64), subsequences=np.array(SUBSEQUENCES, dtype=np.uint64), words=words)
    print("wrote", OUT, words.shape)


if __name__ == "__main__":
    sys.exit(main())
