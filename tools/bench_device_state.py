"""What moving particle state costs a replica batch, through the host calls and through the device-memory calls (pbd_get_attr_device,
pbd_set_attr_device with a replica mask).  ms per step on cfg1 at K = 132 and 1056 and on the 100x100 XPBD cloth at K = 264, in the mode
MODE_AUTO picks, for
    (a) the step alone;
    (b) step + pbd_get_attr of x (every replica, to a host array);
    (c) step + pbd_get_attr_device of x (every replica, to a torch CUDA tensor);
    (d) step + a host restart of 10 % of the replicas: x, v, oldX and lastX of all K read back, the restarted rows patched, all four written;
    (e) step + a masked device restart of the same 10 %: four pbd_set_attr_device calls with the replica mask.
The device calls run on torch's current stream, the engine on a stream of its own, so (c) and (e) pay the two cross-stream event waits a
torch caller pays.  Every variant: warm-up, a probe that sizes the window to at least --window seconds, then the window, timed two ways --
CUDA events on the engine's stream, and a host clock around the window, which ends in a synchronise.  The variants run twice, alternating.
Also the copy kernels alone, 200 of each enqueued behind a spin so that they run back to back: device gets of x, full device sets and
10 % masked device sets, as achieved bandwidth over the algorithmic bytes (DESIGN.md section 3) against the H100 SXM data sheet's 3.35 TB/s.  The card name, power limit and max SM clock are read
in the same run.

    python tools/bench_device_state.py [--out results.json] [--window 0.4] [--quick]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench_batch  # noqa: E402  (card(), the scene builders)
from positionbaseddynamics_b200 import _capi  # noqa: E402

CASES = [("cfg1", 132), ("cfg1", 1056), ("cloth100_xpbd", 264)]
BYTES = {"get": 16 + 12 + 4, "set": 12 + 16 + 16 + 4}  # per particle: DESIGN.md section 3
HBM_TBS = 3.35
ATTRS4 = (_capi.ATTR_X, _capi.ATTR_V, _capi.ATTR_OLDX, _capi.ATTR_LASTX)


class Case:
    def __init__(self, name, k):
        m = bench_batch.model(name)
        self.k, self.n = k, len(m["x0"])
        self.stream = torch.cuda.Stream()  # the engine's own stream; the caller's is torch's current one
        eng = self.eng = _capi.Engine(0, stream=self.stream.cuda_stream)
        eng.set_particles(m["x0"], m["mass"])
        eng.add_flat(m["types"], m["bodies"], m["params"])
        eng.set_groups(m["off"], m["ids"])
        eng.set_params(dt=0.005, sub_steps=m["sub"], max_iter=m["it"])
        eng.set_replicas(k)
        eng.step(1); eng.sync()
        self.active = eng.get_mode()[1]
        self.x0 = eng.get_attr(_capi.ATTR_X).copy()  # the restart state: the batch after one step
        self.v0 = eng.get_attr(_capi.ATTR_V).copy()
        self.restart = np.zeros(k, bool); self.restart[::10] = True  # 10 % of the replicas
        self.host_x = np.empty_like(self.x0)
        self.dx0, self.dv0 = (torch.from_numpy(a.reshape(-1)).cuda() for a in (self.x0, self.v0))
        self.dmask = torch.from_numpy(self.restart).cuda()
        self.dout = torch.empty(k * self.n * 3, device="cuda")
        torch.cuda.synchronize()

    def variant(self, which):
        eng, s = self.eng, torch.cuda.current_stream().cuda_stream
        if which == "a":
            return lambda: eng.step(1)
        if which == "b":
            return lambda: (eng.step(1), eng.get_attr(_capi.ATTR_X, self.host_x))
        if which == "c":
            return lambda: (eng.step(1), eng.get_attr_device(_capi.ATTR_X, self.dout, stream=s))
        if which == "d":
            def host_restart():
                eng.step(1)
                for a, init in zip(ATTRS4, (self.x0, self.v0, self.x0, self.x0)):
                    state = eng.get_attr(a)
                    state[self.restart] = init[self.restart]
                    eng.set_attr(a, state)
            return host_restart
        if which == "e":
            def device_restart():
                eng.step(1)
                for a, src in zip(ATTRS4, (self.dx0, self.dv0, self.dx0, self.dx0)):
                    eng.set_attr_device(a, src, replicas=self.dmask, stream=s)
            return device_restart
        raise ValueError(which)

    def timed(self, fn, window):
        """(event ms, host-clock ms) per call of fn: warm-up, a probe, then a window of at least `window` seconds."""
        for _ in range(3):
            fn()
        self.sync()
        t0 = time.perf_counter()
        for _ in range(5):
            fn()
        self.sync()
        probe = (time.perf_counter() - t0) / 5
        calls = int(min(5000, max(10, window / max(probe, 1e-6))))
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        start.record(self.stream)
        for _ in range(calls):
            fn()
        stop.record(self.stream)
        self.sync()
        wall = (time.perf_counter() - t0) * 1e3 / calls
        return start.elapsed_time(stop) / calls, wall, calls

    def sync(self):
        self.eng.sync()
        torch.cuda.synchronize()

    def close(self):
        self.eng.close()


def copy_bandwidth(c, calls=200, spin=100_000_000):
    """The copy kernels alone (stream=None: on the engine's stream, no cross-stream events), back to back: the engine's stream is held by
    a spin of `spin` cycles (some 50 ms) while the host enqueues `calls` calls, so that the events between them time the kernels and not
    the host's enqueue rate.  enqueue_ms > the spin would mean the host was the limit after all: it is reported next to the times."""
    eng, out = c.eng, {}
    particles = c.k * c.n
    for what, fn, bytes_ in (
            ("get x", lambda: eng.get_attr_device(_capi.ATTR_X, c.dout), BYTES["get"] * particles),
            ("set x", lambda: eng.set_attr_device(_capi.ATTR_X, c.dx0), BYTES["set"] * particles),
            ("set x, 10 % masked", lambda: eng.set_attr_device(_capi.ATTR_X, c.dx0, replicas=c.dmask), BYTES["set"] * c.n * int(c.restart.sum()))):
        for _ in range(3):
            fn()
        c.sync()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(c.stream):
            torch.cuda._sleep(spin)
        t0 = time.perf_counter()
        start.record(c.stream)
        for _ in range(calls):
            fn()
        stop.record(c.stream)
        enqueue_ms = (time.perf_counter() - t0) * 1e3
        c.sync()
        us = start.elapsed_time(stop) * 1e3 / calls
        gbs = bytes_ / (us * 1e-6) * 1e-9
        out[what] = {"us": us, "MB": bytes_ * 1e-6, "GB_s": gbs, "of_hbm": gbs / (HBM_TBS * 1e3), "calls": calls, "enqueue_ms": enqueue_ms}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--window", type=float, default=0.4, help="seconds per timed window")
    ap.add_argument("--quick", action="store_true", help="the smallest case only, short windows (a rehearsal)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_state: no CUDA device")
    res = {"card": bench_batch.card(), "rows": [], "copies": []}
    print("card (name, power limit, max SM clock): %s" % res["card"], flush=True)
    window = 0.05 if a.quick else a.window
    for name, k in CASES[:1] if a.quick else CASES:
        c = Case(name, k)
        row = {"scene": name, "K": k, "particles": k * c.n, "active_mode": c.active, "runs": []}
        for run in range(2):
            times = {}
            for which in "abcde":
                ev, wall, calls = c.timed(c.variant(which), window)
                times[which] = {"event_ms": ev, "wall_ms": wall, "calls": calls}
            row["runs"].append(times)
            print("%-13s K=%5d (%s, %d particles) run %d: " % (name, k, {0: "graph", 1: "resident"}.get(c.active, c.active), k * c.n, run)
                  + " | ".join("(%s) %.3f/%.3f" % (w, t["event_ms"], t["wall_ms"]) for w, t in times.items()) + "  ms/step (events/host clock)", flush=True)
        bw = copy_bandwidth(c)
        res["copies"].append({"scene": name, "K": k, **bw})
        print("   copy kernels: " + " | ".join("%s %.1f us, %.0f GB/s = %.0f %% of 3.35 TB/s (enqueued in %.1f ms)" % (w, v["us"], v["GB_s"], 100 * v["of_hbm"], v["enqueue_ms"])
                                             for w, v in bw.items()), flush=True)
        res["rows"].append(row)
        c.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
