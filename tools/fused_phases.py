"""Per-phase cycle counts of the fused getada3 kernel on the headline workload (diagnostic; needs a GPU)."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    import torch
    from sedumi_b200 import device
    W = bench.load_workload(sys.argv[1] if len(sys.argv) > 1 else bench.HEADLINE)
    hp = device.HotPath(W.S, device=0)
    L = device.lib()
    with torch.cuda.stream(hp.stream()):
        hp.set_scaling(W.d)
        hp.invcholfac()
        for _ in range(3):
            hp.getada()
    hp.sync()
    device.check(L.sb200_ada_fused_profile(hp.ada, 1, None), "profile on")
    reps = 5
    with torch.cuda.stream(hp.stream()):
        for _ in range(reps):
            hp.getada()
    hp.sync()
    out = (C.c_ulonglong * 16)()
    device.check(L.sb200_ada_fused_profile(hp.ada, 0, out), "profile read")
    v = [int(x) for x in out]
    names = ["prologue", "T", "product", "entrywise_W", "dots"]
    tot = sum(v[:5])
    print(json.dumps({"cycles_per_launch": {n: v[i] / reps for i, n in enumerate(names)}, "share": {n: v[i] / tot for i, n in enumerate(names)},
                      "dense_pairs": v[5] / reps, "entrywise_pairs": v[6] / reps,
                      "product_split": {"round1": {"wait_full": v[7] / reps, "issue_next": v[8] / reps, "mma": v[9] / reps},
                                        "later_rounds": {"wait_full": v[11] / reps, "issue_next": v[12] / reps, "mma": v[13] / reps},
                                        "writeback": v[10] / reps}}))


if __name__ == "__main__":
    main()
