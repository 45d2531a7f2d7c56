"""Measures a DER-vs-latency table from ONE sweep over ten latencies (DatasetSweep(..., latencies=...).score_latencies)
against ten single-latency DatasetSweeps built one at a time (construction + score each), on the GPU, and prints one JSON
line (and writes it to --out if given).

Dataset: the 32 seeded synthetic files of tools/sweep_dataset_bench.py (about 4.8 h).  Latencies 0.5, 1.0, ..., 5.0 s;
T in {16, 256} trials.  Reported, in one process, with the card's name and power limit read in the same call:

    latency_sweep   construction time and resident bytes of the one sweep over all ten latencies, then per T the host
                    clock and the device time (CUDA events around the launches) of score_latencies, and the trial groups
                    (launches) it makes
    per_latency     per T: the ten DatasetSweeps at one latency each, each constructed and scored in turn (one alive at a
                    time), summed; their construction time is counted once, in the first T's row
    components_equal  every (latency, file, trial) component of the two legs equal bit for bit (exit status 1 otherwise)

--vad does the same for VoiceActivitySweep (tau_active trials).

    python tools/latency_sweep_bench.py [--files 32] [--vad] [--out /tmp/latency_sweep_bench.json]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from diart_b200 import blocks, models  # noqa: E402
from diart_b200.tune import DatasetSweep, VoiceActivitySweep, trial_groups  # noqa: E402
from sweep_bench import card, trials as diarization_trials  # noqa: E402
from sweep_dataset_bench import make_dataset  # noqa: E402
from vad_sweep_bench import trials as vad_trials  # noqa: E402

LATENCIES = [0.5 * i for i in range(1, 11)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=32)
    ap.add_argument("--vad", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no GPU: nothing to measure")
    from oracle import nets

    dev = torch.device("cuda", 0)
    seg_state, emb_state = nets.make_segmentation().state_dict(), nets.make_embedding().state_dict()

    def config(latency):
        seg = models.SegmentationModel(models.B200SegmentationLoader(seg_state))
        if args.vad:
            return blocks.VoiceActivityDetectionConfig(segmentation=seg, device=dev, latency=latency)
        emb = models.EmbeddingModel(models.B200EmbeddingLoader(emb_state))
        return blocks.SpeakerDiarizationConfig(segmentation=seg, embedding=emb, device=dev, latency=latency)

    kind = VoiceActivitySweep if args.vad else DatasetSweep
    make_trials = vad_trials if args.vad else diarization_trials
    result = {"card": card(), "sweep": kind.__name__, "latencies": LATENCIES}
    files = make_dataset(args.files)
    result["files"] = len(files)
    result["audio_hours"] = sum(len(x) for _, x, _ in files) / 16000 / 3600
    kind(config(0.5), files[:2], latencies=LATENCIES).score_latencies(make_trials(4))   # warm-up: handles, attributes

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ds = kind(config(0.5), files, latencies=LATENCIES)
    torch.cuda.synchronize()
    nv = ds.units.num_virtual(range(len(LATENCIES)))
    result["latency_sweep"] = {"construct_s": time.perf_counter() - t0, "resident_gb": ds.resident_bytes / 1e9,
                               "real_chunks": ds.num_chunks, "virtual_chunks": nv, "units": len(ds.offsets) - 1}
    ds.score_latencies(make_trials(4))                                 # warm-up of the dataset-sized buffers
    got, rows = {}, {}
    for T in (16, 256):
        tr = make_trials(T)
        best_call, best_dev = None, None
        for _ in range(2):
            t0 = time.perf_counter()
            got[T] = ds.score_latencies(tr)
            call = time.perf_counter() - t0
            best_call = call if best_call is None else min(best_call, call)
            best_dev = ds.timing["score"] if best_dev is None else min(best_dev, ds.timing["score"])
        groups = trial_groups(T, nv)
        rows[T] = {"score_latencies_call_s": best_call, "score_latencies_device_s": best_dev, "launches": len(groups),
                   "trials_per_launch": groups[0].stop - groups[0].start}
    del ds
    gc.collect()

    # the same table from ten single-latency sweeps, one alive at a time
    equal = True
    construct = 0.0
    for T in rows:
        rows[T].update({"per_latency_construct_s": 0.0, "per_latency_score_s": 0.0, "per_latency_score_device_s": 0.0,
                        "per_latency_launches": 0})
    for lat in LATENCIES:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        one = kind(config(lat), files)
        torch.cuda.synchronize()
        construct += time.perf_counter() - t0
        for T in rows:
            t0 = time.perf_counter()
            per_file, total = one.score(make_trials(T))
            rows[T]["per_latency_score_s"] += time.perf_counter() - t0
            rows[T]["per_latency_score_device_s"] += one.timing["score"]
            rows[T]["per_latency_launches"] += len(trial_groups(T, one.num_chunks))
            g_per_file, g_total = got[T][lat]
            same = all(np.array_equal(a.as_array(), b.as_array()) for a, b in zip(g_per_file, per_file)) and \
                np.array_equal(g_total.as_array(), total.as_array())
            rows[T].setdefault("components_equal", True)
            rows[T]["components_equal"] &= bool(same)
            equal &= bool(same)
        del one
        gc.collect()
    first = True
    for T in rows:
        r = rows[T]
        r["per_latency_construct_s"] = construct if first else 0.0
        first = False
        r["per_latency_total_s"] = r["per_latency_construct_s"] + r["per_latency_score_s"]
        r["score_speedup_device"] = r["per_latency_score_device_s"] / r["score_latencies_device_s"]
        metric = "detection_error_rate" if args.vad else "der"
        r["best_per_latency"] = {str(lat): float(getattr(got[T][lat][1], metric).min()) for lat in LATENCIES}
    result["per_latency_construct_s"] = construct
    result["trials"] = rows
    result["components_equal"] = equal
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not equal:
        sys.exit("the components of the sweep over ten latencies differ from the single-latency sweeps'")


if __name__ == "__main__":
    main()
