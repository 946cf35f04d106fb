"""Measured FP64 peaks of GPU 0: the vector pipe (DFMA chains, world_b200_fp64_peak) and the tensor cores
(mma.m16n8k4.f64 chains, world_b200_fp64_tensor_peak), in one process and on the same card.  Prints one
JSON line.  Development aid: Harvest's filter bank (band_fir_events_kernel) runs on the tensor cores."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from world_b200.api import World


def main():
    w = World(device=0)
    res = {"device": torch.cuda.get_device_name(0), "runs": []}
    for _ in range(3):   # alternated, so that clock drift shows up in both figures
        res["runs"].append({"dfma_tflops": w.fp64_peak(), "dmma_tflops": w.fp64_tensor_peak()})
    dfma = max(r["dfma_tflops"] for r in res["runs"])
    dmma = max(r["dmma_tflops"] for r in res["runs"])
    res.update(dfma_tflops=dfma, dmma_tflops=dmma, dmma_over_dfma=dmma / dfma)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
