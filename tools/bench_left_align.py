"""Bench line of `variants --vcf --reference --left-align` (K15d, K15i; an extension): BASELINE.json configs[3]
(`cfg4_5Mb_200x`, as bench.py builds it), bench.py's single-GPU step, then the left-alignment kernels over its batch
against the config-4 contig with a homopolymer or dinucleotide repeat planted every 997 bases.

    python tools/bench_left_align.py [--steps K] [--warmup W]      # one JSON line on stdout

The timed step is bench.py's.  On top of bench.py's fields the line carries:
  `left_align_ms`  K15d with its regrouping (engine.left_align_deletions over K7's groups), K15i over the step's
                   insertion rows with its zeroed H (engine.left_align_insertions), K7 with its grouping
                   (engine._deletion_groups) and K6r's two passes, in 7 alternating rounds of 20 launches;
  `e2e_vcf`        variants_vcf(path, reference=fa, left_align=True) against the same call without it on a 10^6-read
                   BAM, best of 3, alternating;
  `gpu`            the card's name and power limit, read in the same run;
  `parity`         the sha256 of K15d's moved keys and of K15i's H and moved slots equal those of the oracle's per-base
                   loops (oracle/py_laoracle.py), and the step's calls equal the C oracle's.
Writes nothing into the tree."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from bench_fastq import alternate  # noqa: E402
from bench_variants_ref import contig_text, gpu_info  # noqa: E402

WORKLOAD = "cfg4_5Mb_200x"


def planted(text, seed=4, every=997):
    """The contig's text with a 12-base homopolymer or dinucleotide repeat every `every` bases."""
    out = list(text)
    rng = np.random.default_rng(seed)
    for at in range(50, len(out) - 20, every):
        a, b = "ACGT"[rng.integers(4)], "ACGT"[rng.integers(4)]
        out[at:at + 12] = list(a * 12 if rng.random() < 0.5 else (a + b) * 6)
    return "".join(out)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def oracle_moves(batch, codes, events, ev_slot, ev_len):
    """(sorted unique moved deletion keys, moved insertion slots, H) by the oracle's per-base loops."""
    from kindel_b200.insertions import decode_events
    from oracle import py_laoracle as LO

    letters = "".join("ACGTN"[c] for c in codes.tolist())
    s0 = int(batch.contig_slot[0])
    keys = sorted({((s0 + LO.left_deletion(letters[s0:r + n], r - s0, n)) << 28) | n
                   for r, n in zip(ev_slot.tolist(), ev_len.tolist())})
    slots = np.empty(len(events), dtype=np.int64)
    for i, (row, t) in enumerate(zip(events.tolist(), decode_events(batch, events))):
        slots[i] = s0 + LO.left_insertion(letters[s0:row[0]], row[0] - s0, t)[0]
    hist = np.bincount(slots, minlength=int(batch.n_slots)).astype(np.int32)
    return np.array(keys, dtype=np.int64), slots, hist


def e2e_vcf(rounds=3):
    from kindel_b200 import kindel as K
    from kindel_b200 import synth

    sub = synth.simple_reads(4, [750_000], 200)  # 10^6 reads, as bench.py's host block
    with tempfile.TemporaryDirectory() as tmp:
        path, fa = os.path.join(tmp, "slice.bam"), os.path.join(tmp, "slice.fa")
        synth.write_simple_bam(path, sub)
        with open(fa, "w") as fh:
            fh.write(">ctg0\n" + planted(contig_text(4, 750_000)) + "\n")
        K.variants_vcf(path, reference=fa, left_align=True), K.variants_vcf(path, reference=fa)  # warm
        best = {"left_align": None, "reference": None}
        for _ in range(rounds):
            for key, fn in (("left_align", lambda: K.variants_vcf(path, reference=fa, left_align=True)),
                            ("reference", lambda: K.variants_vcf(path, reference=fa))):
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                best[key] = dt if best[key] is None or dt < best[key] else best[key]
    return {"left_align_s": best["left_align"], "reference_s": best["reference"], "reads": int(sub.n_reads),
            "note": "variants_vcf(path, reference=fa, left_align=True) vs variants_vcf(path, reference=fa), best of %d, "
                    "alternating" % rounds}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args(argv)

    import torch

    from kindel_b200 import engine
    from kindel_b200.reference import load_reference
    from oracle import coracle

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = gpu_info()
    batch = bench.gen_reads(WORKLOAD)
    n_slots = batch.n_slots
    db = engine.upload(batch, dev)
    table = engine.CountTable(n_slots, dev)
    calls_buf = torch.empty(n_slots, dtype=torch.uint8, device=dev)

    def step(timers=None):
        if timers:
            timers[0].record()
        engine.pileup(db, check=False, table=table)
        if timers:
            timers[1].record()
        out = engine.vote(table.t, 1, out=calls_buf)
        if timers:
            timers[2].record()
        return out

    tm = bench.time_steps(step, args.steps, args.warmup, torch, None, 1, dev)
    calls = tm["out"].cpu().numpy()

    with tempfile.TemporaryDirectory() as tmp:
        fa = os.path.join(tmp, "cfg4.fa")
        with open(fa, "w") as fh:
            fh.write(">%s\n%s\n" % (batch.contig_names[0], planted(contig_text(4, int(batch.contig_len[0])))))
        ref = load_reference(fa, batch)
    t_ref = torch.from_numpy(ref.codes).to(dev)
    _, events = engine.pileup(db)
    key, cnt = engine._deletion_groups(db)
    cs = db.tensors["contig_slot"]
    a, r = 1, 0.01
    timing = alternate((
        ("k15d_left_align_deletions", lambda: engine.left_align_deletions(key, cnt, t_ref, cs, batch.n_contigs)),
        ("k15i_left_align_insertions", lambda: engine.left_align_insertions(db, events, t_ref)),
        ("k7_deletion_groups", lambda: engine._deletion_groups(db)),
        ("k6r_variants_ref", lambda: engine.variant_sites_ref(table.t, batch.contig_slot, batch.contig_len, t_ref,
                                                              a, r))), torch)
    moved, _ = engine.left_align_deletions(key, cnt, t_ref, cs, batch.n_contigs)
    norm_slot, _, hist = engine.left_align_insertions(db, events, t_ref)
    host_events = events.cpu().numpy()
    timing.update(deletion_groups=int(key.numel()), insertion_rows=int(host_events.shape[0]),
                  rows_moved=int((norm_slot.cpu().numpy() != host_events[:, 0]).sum()),
                  note="k15d includes torch.unique and the count sum of the regrouping; k7 its read-back of the event "
                       "total and its grouping; k6r its read-back of the site total and the copy of the sites")
    e2e = e2e_vcf()

    ev_slot, ev_len = engine.deletion_events(db)
    want_keys, want_slots, want_hist = oracle_moves(batch, ref.codes, host_events, ev_slot.cpu().numpy(),
                                                    ev_len.cpu().numpy())
    parity_keys = _sha(moved.cpu().numpy()) == _sha(want_keys)
    parity_hist = _sha(hist.cpu().numpy()) == _sha(want_hist)
    parity_slots = _sha(norm_slot.cpu().numpy()) == _sha(want_slots)
    want_calls = coracle.vote(coracle.pileup(batch)[0], 1)
    parity = bool(parity_keys and parity_hist and parity_slots and np.array_equal(calls, want_calls))
    ms_per_step = tm["total_ms"] / tm["reps"]
    line = {
        "metric": bench.METRIC, "value": batch.aligned_bases / (ms_per_step * 1e-3), "unit": bench.UNIT, "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": parity, "parity_detail": {"k15d_keys_sha256": bool(parity_keys), "k15i_hist_sha256": bool(parity_hist),
                                            "k15i_slots_sha256": bool(parity_slots)},
        "config": {"workload": WORKLOAD, "reads_per_rank": int(batch.n_reads),
                   "complex_reads_per_rank": int(batch.n_complex), "aligned_bases_total": int(batch.aligned_bases),
                   "tool": "tools/bench_left_align.py",
                   "parity_oracle": "oracle/py_laoracle.py's per-base loops over K7's events and the step's insertion "
                                    "rows; the step's calls against oracle/kindel_oracle.c"},
        "gpu": gpu, "left_align_ms": timing, "e2e_vcf": e2e, "e2e": None,
    }
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
