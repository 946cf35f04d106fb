"""GPU experiment: host pipeline (world_b200_analyze_host / _coded_host) versus its outer / sub chunk sizes.
Usage (on a GPU machine):  python tools/exp_host_chunks.py [n_utts] > host_chunks.txt"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
from world_b200.api import World, F0_HARVEST  # noqa: E402
from synth import synth_batch  # noqa: E402


def main():
    U = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    fs, n = 16000, 160000
    dev = torch.device("cuda:0")
    w = World(device=0)
    L = w.frames(fs, n)
    bins = 513
    xh = torch.empty((U, n), dtype=torch.float64, pin_memory=True)
    for u0 in range(0, U, 64):
        u1 = min(U, u0 + 64)
        xh[u0:u1].copy_(synth_batch(range(u0 + 1, u1 + 1), fs, n, device=dev))
    ph = torch.empty((U, n), dtype=torch.int16, pin_memory=True)
    ph.copy_((xh * 32767.0).round().to(torch.int16))
    th = torch.empty((U, L), dtype=torch.float64, pin_memory=True)
    fh = torch.empty((U, L), dtype=torch.float64, pin_memory=True)
    sph = torch.empty((U, L, bins), dtype=torch.float64, pin_memory=True)
    aph = torch.empty((U, L, bins), dtype=torch.float64, pin_memory=True)
    csh = torch.empty((U, L, 60), dtype=torch.float64, pin_memory=True)
    cah = torch.empty((U, L, 1), dtype=torch.float64, pin_memory=True)
    ao = w.analysis_option(fs, F0_HARVEST)
    w.set_scratch_budget(64 << 30)

    def raw():
        w.analyze_host(xh, fs, ao, time_axis=th, f0=fh, spectrogram=sph, aperiodicity=aph, f0_stride=L)

    def coded():
        w.analyze_coded_host(ph, 16, fs, ao, 60, time_axis=th, f0=fh, coded_sp=csh, coded_ap=cah, f0_stride=L)

    raw(); coded()
    for outer, sub in ((256, 64), (256, 128), (512, 128), (1024, 128), (96, 96)):
        os.environ["WB_HOST_CHUNK"], os.environ["WB_HOST_SUB"] = str(outer), str(sub)
        w.trim()
        res = []
        for fn in (raw, coded):
            fn()
            ts = []
            for _ in range(2):
                t0 = time.perf_counter(); fn(); ts.append((time.perf_counter() - t0) * 1e3)
            res.append(ts)
        print(f"outer {outer:5d} sub {sub:4d}  raw ms {res[0][0]:8.1f} {res[0][1]:8.1f}   coded ms {res[1][0]:8.1f} {res[1][1]:8.1f}", flush=True)
    # one traced call each at the defaults
    os.environ.pop("WB_HOST_CHUNK"); os.environ.pop("WB_HOST_SUB")
    w.trim(); raw(); coded()
    os.environ["WB_HOST_TRACE"] = "1"
    sys.stderr.write("---- trace raw\n"); sys.stderr.flush(); raw()
    sys.stderr.write("---- trace coded\n"); sys.stderr.flush(); coded()


if __name__ == "__main__":
    main()
