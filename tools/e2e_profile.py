"""cProfile of the host thread while host-resident batches stream through the device
(where does the host time per slice go?).  On a GPU machine: python tools/e2e_profile.py"""
import cProfile
import os
import pstats
import sys
import time
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchio_b200 as tio  # noqa: E402
from torchio_b200 import parallel  # noqa: E402

B, S = 32, 256
parallel.bind_to_gpu_numa(0)
with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    pipe = tio.Compose([
        tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)), tio.ElasticDeformation(), tio.BiasField(),
        tio.Blur(std=(0, 2)), tio.Noise(std=(0, 0.25)), tio.Gamma(log_gamma=(-0.3, 0.3))], copy=False)
host = torch.rand((B, 1, S, S, S)).pin_memory()
affines = [tio.AffineMatrix() for _ in range(B)]
pipe.chunk_bytes = int(os.environ.get("CHUNK_MB", "128")) << 20


def batches(n):
    for _ in range(n):
        yield tio.SubjectsBatch({"t1": tio.ImagesBatch(host, list(affines))})


with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    for _ in pipe.stream(batches(4), depth=1):
        pass
    torch.cuda.synchronize()
    prof = cProfile.Profile()
    t0 = time.perf_counter()
    prof.enable()
    for _ in pipe.stream(batches(6), depth=1):
        pass
    prof.disable()
    torch.cuda.synchronize()
    print("ms/step", (time.perf_counter() - t0) * 1e3 / 6)
st = pstats.Stats(prof)
st.sort_stats("cumulative").print_stats(45)
st.sort_stats("tottime").print_stats(30)
