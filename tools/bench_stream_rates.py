"""What a FaceAnaStreams call costs when cameras run at their own frame rates (submit(frames, streams=...)): S streams of
the 1080p 4-face scene, faces jittered on every frame so that the detector runs on every frame, pinned host frames in,
host results out, two calls in flight.

    python tools/bench_stream_rates.py [--streams 16] [--batches 12] [--rounds 5]

Modes, each on its own object, alternated over --rounds rounds (the order rotates every round), median of the rounds:
  lockstep    FaceAnaStreams(n_streams=S): all S streams every call
  mixed       FaceAnaStreams(n_streams=S): S/2 streams on every call, the other S/2 on every other call, each call's
              order shuffled; ms per S-frame call and per S/2-frame call, and frames/s overall
  subset      FaceAnaStreams(n_streams=S): S/2 of the S streams on every call, shuffled
  half        FaceAnaStreams(n_streams=S/2): all of its streams every call
A call's time is the host interval between the return of its collect() and that of the previous call's, with the next
call already submitted: with two calls in flight, the time the pipeline spends on that call.  Every batch size a timed
window meets is warmed up first.  The GPU name and power limit are read in the same run."""
import json
import os
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402


class Feed:
    """One FaceAnaStreams object and each stream's position in its clip."""

    def __init__(self, fa, seqs):
        self.fa, self.seqs = fa, seqs
        self.pos = [0] * len(seqs)

    def submit(self, streams):
        batch = []
        for s in streams:
            batch.append(self.seqs[s][self.pos[s] % len(self.seqs[s])])
            self.pos[s] += 1
        self.fa.submit(batch, streams=streams)

    def window(self, calls):
        """Runs the calls with two in flight; (total seconds, per-call seconds of calls 1..)."""
        import torch
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        self.submit(calls[0])
        stamps = []
        for c in calls[1:]:
            self.submit(c)
            self.fa.collect()
            stamps.append(time.perf_counter())
        self.fa.collect()
        stamps.append(time.perf_counter())
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        return total, list(np.diff(stamps))


def schedules(S, batches, rng):
    full, fast, slow = list(range(S)), list(range(0, S, 2)), list(range(1, S, 2))

    def shuffled(x):
        return [int(v) for v in rng.permutation(x)]
    return {
        "lockstep": [full] * batches,
        # even calls: every stream; odd calls: the fast half only
        "mixed": [shuffled(fast + slow) if t % 2 == 0 else shuffled(fast) for t in range(batches)],
        "subset": [shuffled(fast) for _ in range(batches)],
        "half": [list(range(S // 2))] * batches,
    }


def main():
    import torch
    import frames
    from Skps import FaceAnaStreams
    from bench_streams import gpu_info, make_streams
    a = sys.argv[1:]

    def opt(name, default):
        return a[a.index(name) + 1] if name in a else default
    S, batches, rounds = int(opt("--streams", 16)), int(opt("--batches", 12)), int(opt("--rounds", 5))
    assert S % 2 == 0 and batches % 2 == 0, "--streams and --batches must be even"
    print(json.dumps(gpu_info(torch)))
    sys.stdout.flush()
    seqs = make_streams(torch, frames, frames.frame_1080p, S, length=6)
    H, W = seqs[0][0].shape[:2]
    top_k = 4
    feeds = {k: Feed(FaceAnaStreams(n_streams=S, top_k=top_k, max_frame_hw=(H, W)), seqs)
             for k in ("lockstep", "mixed", "subset")}
    feeds["half"] = Feed(FaceAnaStreams(n_streams=S // 2, top_k=top_k, max_frame_hw=(H, W)), seqs[:S // 2])
    rng = np.random.default_rng(0)
    for k, f in feeds.items():             # every batch size of the timed windows (S and S/2 frames), twice in flight
        f.window(schedules(S, 6, rng)[k])
    modes = list(feeds)
    totals = {k: [] for k in modes}
    per_call = {k: {} for k in modes}      # frames per call -> per-round medians
    for r in range(rounds):
        plan = schedules(S, batches, rng)
        for k in modes[r % len(modes):] + modes[:r % len(modes)]:
            total, dts = feeds[k].window(plan[k])
            totals[k].append(total)
            by_n = {}
            for c, dt in zip(plan[k][1:], dts):
                by_n.setdefault(len(c), []).append(dt)
            for n, v in by_n.items():
                per_call[k].setdefault(n, []).append(float(np.median(v)))
    frames_per_window = {k: sum(len(c) for c in schedules(S, batches, np.random.default_rng(0))[k]) for k in modes}
    out = {"config": "1080p_4faces", "n_streams": S, "top_k": top_k, "calls_per_window": batches, "rounds": rounds,
           "detector": "every frame (faces jittered every frame)"}
    for k in modes:
        med = float(np.median(totals[k]))
        out[k] = {"ms_per_call": 1e3 * med / batches, "frames_per_s": frames_per_window[k] / med,
                  "ms_per_call_by_frames": {str(n): 1e3 * float(np.median(v)) for n, v in sorted(per_call[k].items())},
                  "ms_per_call_rounds": [1e3 * t / batches for t in totals[k]]}
    out["api"] = "FaceAnaStreams.submit(frames, streams=...)/collect, pinned host frames, host results, 2 calls in flight"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
