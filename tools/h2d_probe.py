"""Pinned host<->device copy bandwidth of the machine (what bounds the e2e arm), and the CPU quota the process sees."""
import torch, time
for mb in (64, 359):
    h = torch.empty(mb << 20, dtype=torch.uint8).pin_memory()
    d = torch.empty(mb << 20, dtype=torch.uint8, device="cuda")
    for direction in ("h2d", "d2h"):
        best = 1e9
        for _ in range(5):
            torch.cuda.synchronize(); t0 = time.perf_counter()
            (d.copy_(h, non_blocking=True) if direction == "h2d" else h.copy_(d, non_blocking=True))
            torch.cuda.synchronize(); best = min(best, time.perf_counter() - t0)
        print(direction, mb, "MB", round(mb / 1024 / best, 2), "GB/s", round(best * 1e3, 2), "ms")
for f in ("/sys/fs/cgroup/cpu.max", "/proc/loadavg"):
    try:
        print(f, open(f).read().strip())
    except Exception as ex:
        print(f, ex)
import os; print("nproc", len(os.sched_getaffinity(0)))
