"""How the measurement tools take a time and read the card, so that two numbers from two tools were taken the same way.

    device_ms(fn, reps, warmup)   CUDA events around `reps` calls of fn, after `warmup` calls and a synchronise
    host_ms(fn, reps=..., ...)    the host clock around `reps` calls of fn, or around as many as fill `min_s` seconds
    card(), card_line()           the current device's name, power limit and max SM clock, read with nvidia-smi

A tool run as `python tools/x.py` has tools/ first on sys.path, so `import devtime` finds this module.  Each tool passes
its own warm-up and rep counts: they are what keeps its numbers comparable with the ones already published.
"""
import subprocess
import time

import torch


def device_ms(fn, reps, warmup):
    """Milliseconds per call of fn on the current stream: `warmup` calls, a device synchronise, then a CUDA event pair
    around `reps` calls.  There is no host-clock fallback: without a CUDA device this raises."""
    if not torch.cuda.is_available():
        raise RuntimeError("device_ms needs a CUDA device")
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def host_ms(fn, reps=None, warmup=1, min_s=None):
    """Host wall-clock milliseconds per call of fn after `warmup` calls: over exactly `reps` calls, or, with `min_s`,
    over as many calls as it takes for the clock to pass min_s seconds.  fn must finish its own work (numpy, cv2, or a
    device synchronise) before it returns."""
    if (reps is None) == (min_s is None):
        raise ValueError("host_ms takes either reps or min_s")
    for _ in range(warmup):
        fn()
    t0 = time.perf_counter()
    if reps is not None:
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) * 1e3 / reps
    n = 0
    while True:
        fn()
        n += 1
        dt = time.perf_counter() - t0
        if dt >= min_s:
            return dt * 1e3 / n


def card():
    """{name, power_limit_w, sm_clock_max_mhz} of the current CUDA device, from a read-only nvidia-smi query.  The
    device is named by its UUID, so the reading is the card the tool runs on whatever CUDA_VISIBLE_DEVICES says
    (without a CUDA device, nvidia-smi's first card).  If the query fails, every value is the error text: a number is
    still worth printing, beside what went wrong."""
    try:
        ids = [f"--id=GPU-{torch.cuda.get_device_properties(None).uuid}"] if torch.cuda.is_available() else []
        q = subprocess.run(["nvidia-smi", *ids, "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30, check=True)
        name, power, clock = (s.strip() for s in q.stdout.splitlines()[0].split(","))
        return dict(name=name, power_limit_w=float(power), sm_clock_max_mhz=float(clock))
    except Exception as e:                                 # noqa: BLE001
        err = " ".join(f"card not read: {e} {getattr(e, 'stderr', None) or ''}".split())
        return dict(name=err, power_limit_w=err, sm_clock_max_mhz=err)


def card_line(c=None):
    """One line for a text tool to print beside its numbers; `c` is a card() reading to format, by default a new one."""
    c = c or card()
    if isinstance(c["power_limit_w"], str):
        return c["name"]
    return f"{c['name']}, power limit {c['power_limit_w']:g} W, max SM clock {c['sm_clock_max_mhz']:g} MHz"
