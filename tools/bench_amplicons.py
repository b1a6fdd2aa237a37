"""Bench line of the per-amplicon report (`kindel amplicons`, K12 and K12d; an extension): bench.py's single-GPU step
over BASELINE.json configs[3] (`cfg4_5Mb_200x`, as bench.py builds it), then K12, the count of its labels and K12d
over two workloads of that size, each with synth.tiled_scheme's rows written as a named BED (synth.named_scheme_bed:
`amp_<k>_LEFT` / `amp_<k>_RIGHT`, pools alternating):

  cfg4       the step's batch (1 % complex reads); uniform read starts put only a fraction of the reads in a primer
  amplicon   synth.amplicon_reads: every read starts at a left primer or ends at a right one

    python tools/bench_amplicons.py [--steps K] [--warmup W]      # one JSON line on stdout

On top of bench.py's fields the line carries, per workload (`amplicons_ms`):
  `ms`        K12 alone (kdl_amplicons_assign into preallocated labels), the count of the labels per class and amplicon
              (kindel.amplicon_label_counts, and one torch.bincount of all labels beside it), K12d alone
              (kdl_amplicons_depth into preallocated stats) and K0 + K1 (the pileup into a reused table) for scale, in
              7 alternating rounds of 20 launches;
  reads per label class, amplicons, and the bytes K12 and K12d read;
  `parity`    the labels have the sha256 of oracle/py_aoracle.py's labels_of_batch, and K12d's stats the sha256 of its
              insert_stats over the same (primer-masked) count table.
`e2e_amplicons` times kindel.amplicons(path, bed) against bam_to_consensus(path, primers=bed) on a 10^6-read amplicon
BAM, best of 3, alternating; `gpu` is the card's name and power limit, read in the same run.  Writes nothing into the
tree."""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from bench_fastq import alternate  # noqa: E402
from bench_variants_ref import gpu_info  # noqa: E402

WORKLOAD = "cfg4_5Mb_200x"
SCHEME_SEED = 1


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def tiled_named_rows(rows):
    """tiled_scheme's rows as the oracle's (chrom, start, end, amplicon, side), named as named_scheme_bed names them."""
    out, k_of = [], {}
    for i in range(0, len(rows), 2):
        (c, a, b), (_, x, y) = rows[i], rows[i + 1]
        k = k_of.get(c, 0)
        k_of[c] = k + 1
        out += [(c, a, b, "amp_%d" % k, "L"), (c, x, y, "amp_%d" % k, "R")]
    return out


def amplicon_workload(batch, rows, torch, dev):
    from kindel_b200 import _ffi, engine, primers, synth
    from kindel_b200.kindel import amplicon_label_counts
    from oracle import py_aoracle

    lib = _ffi.load()
    scheme = primers.read_scheme(synth.named_scheme_bed(rows).encode(), "scheme.bed")
    arrays = primers.amplicon_arrays(scheme, batch.contig_names, batch.contig_len)
    plain = engine.upload(batch, dev)
    table = engine.CountTable(batch.n_slots, dev)
    masked = engine.mask_primers(engine.upload(batch, dev),
                                 primers.primer_arrays(scheme.primers, batch.contig_names, batch.contig_len))
    counts = engine.pileup(masked)[0]
    labels = engine.assign_amplicons(masked, arrays)
    stats = engine.amplicon_depth(counts, arrays, 20, batch.contig_slot, batch.contig_len)
    st = int(torch.cuda.current_stream(dev).cuda_stream)
    a, keep = engine._amplicons_on(arrays, dev)
    slot, length, n_contigs = engine._device_layout(batch.contig_slot, batch.contig_len, dev)
    lab_buf = torch.empty_like(labels)
    stats_buf = torch.empty_like(stats)
    n_amp = arrays.n_amplicons

    def k12():
        lib.kdl_amplicons_assign(C.byref(masked.struct), C.byref(a), lab_buf.data_ptr(), st)

    def k12d():
        lib.kdl_amplicons_depth(counts.data_ptr(), batch.n_slots, slot.data_ptr(), length.data_ptr(), n_contigs,
                                C.byref(a), 20, stats_buf.data_ptr(), st)

    timing = alternate((("k0_k1_pileup", lambda: engine.pileup(plain, check=False, table=table)),
                        ("k12_assign", k12), ("label_counts", lambda: amplicon_label_counts(labels, n_amp)),
                        ("bincount_all", lambda: torch.bincount(labels.long() + 3, minlength=n_amp + 3)),
                        ("k12d_depth", k12d)), torch)
    same = bool(torch.equal(lab_buf, labels) and torch.equal(stats_buf, stats) and torch.equal(
        amplicon_label_counts(labels, n_amp), torch.bincount(labels.long() + 3, minlength=n_amp + 3)))
    got = labels.cpu().numpy().astype(np.int64)
    cls = {k: int((got == v).sum()) for k, v in (("unprimed", -1), ("mispaired", -2), ("ambiguous", -3))}
    cx_words = int(sum(2 + int(batch.cig_off[r + 1] - batch.cig_off[r]) for r in np.asarray(batch.complex_idx)))
    ins = int((arrays.insert_end - arrays.insert_start).astype(np.int64).sum())
    timing.update(reads=int(batch.n_reads), assigned=int((got >= 0).sum()), amplicons=n_amp, **cls,
                  k12_bytes_read=int(12 * batch.n_reads + 4 * cx_words), k12_bytes_written=int(4 * batch.n_reads),
                  k12d_bytes_read=int(16 * ins), segments=int(arrays.left_at.shape[0] + arrays.right_at.shape[0]),
                  note="k12_assign / k12d_depth: the entry points over preallocated outputs, no read-back; label_counts: "
                       "kindel.amplicon_label_counts (three class reductions + bincount of the assigned labels); "
                       "bincount_all: one torch.bincount of all labels, for comparison; k0_k1_pileup: engine.pileup "
                       "into a reused CountTable")
    print("amplicons: timed %d reads, checking against the oracle" % batch.n_reads, file=sys.stderr, flush=True)
    nrows = tiled_named_rows(rows)
    want = py_aoracle.labels_of_batch(batch, nrows)
    names = list(batch.contig_names)
    want_stats = np.array(py_aoracle.insert_stats(counts.cpu().numpy(), batch.contig_slot, names,
                                                  py_aoracle.amplicon_table(nrows, names), 20), dtype=np.int64)
    got_stats = stats.cpu().numpy().astype(np.int64).reshape(-1, 3)
    detail = {"labels_sha256": sha(got), "oracle_labels_sha256": sha(want), "stats_sha256": sha(got_stats),
              "oracle_stats_sha256": sha(want_stats)}
    detail["parity"] = bool(sha(got) == sha(want) and sha(got_stats) == sha(want_stats) and same)
    del keep
    return timing, detail


def e2e(rounds=3):
    from kindel_b200 import kindel as K
    from kindel_b200 import synth

    sub, rows = synth.amplicon_reads(4, 750_000, 200)  # 10^6 reads, as bench.py's host block
    with tempfile.TemporaryDirectory() as tmp:
        path, bed = os.path.join(tmp, "amp.bam"), os.path.join(tmp, "scheme.bed")
        synth.write_simple_bam(path, sub)
        with open(bed, "w") as fh:
            fh.write(synth.named_scheme_bed(rows))
        K.amplicons(path, bed), K.bam_to_consensus(path, primers=bed)  # warm
        best = {"amplicons": None, "consensus_primers": None}
        for _ in range(rounds):
            for key, fn in (("amplicons", lambda: K.amplicons(path, bed)),
                            ("consensus_primers", lambda: K.bam_to_consensus(path, primers=bed))):
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                best[key] = dt if best[key] is None or dt < best[key] else best[key]
    return {"amplicons_s": best["amplicons"], "consensus_primers_s": best["consensus_primers"],
            "reads": int(sub.n_reads), "amplicons": len(rows) // 2,
            "note": "kindel.amplicons(path, bed) vs bam_to_consensus(path, primers=bed), best of %d, alternating" % rounds}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args(argv)

    import torch

    from kindel_b200 import engine, synth

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = gpu_info()
    batch = bench.gen_reads(WORKLOAD)
    db = engine.upload(batch, dev)
    table = engine.CountTable(batch.n_slots, dev)
    calls_buf = torch.empty(batch.n_slots, dtype=torch.uint8, device=dev)

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
    del db, table
    out = {}
    rows = synth.tiled_scheme(SCHEME_SEED, batch.contig_names, batch.contig_len)
    print("step timed: %.4f ms" % (tm["total_ms"] / tm["reps"]), file=sys.stderr, flush=True)
    out["cfg4"] = amplicon_workload(batch, rows, torch, dev)
    cfg = dict(reads=int(batch.n_reads), complex=int(batch.n_complex), aligned=int(batch.aligned_bases))
    del batch
    torch.cuda.empty_cache()
    amp, amp_rows = synth.amplicon_reads(4, 5_000_000, 200)
    out["amplicon"] = amplicon_workload(amp, amp_rows, torch, dev)
    aligned = int(amp.aligned_bases)
    del amp
    torch.cuda.empty_cache()
    print("timing kindel.amplicons", file=sys.stderr, flush=True)
    e2e_line = e2e()
    parity = all(v[1]["parity"] for v in out.values())
    ms_per_step = tm["total_ms"] / tm["reps"]
    line = {
        "metric": bench.METRIC, "value": cfg["aligned"] / (ms_per_step * 1e-3), "unit": bench.UNIT,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": parity, "parity_detail": {k: v[1] for k, v in out.items()},
        "config": {"workload": WORKLOAD, "reads_per_rank": cfg["reads"], "complex_reads_per_rank": cfg["complex"],
                   "aligned_bases_total": cfg["aligned"], "amplicon_aligned_bases": aligned,
                   "scheme_seed": SCHEME_SEED, "tool": "tools/bench_amplicons.py",
                   "parity_oracle": "oracle/py_aoracle.py (labels_of_batch, insert_stats)"},
        "gpu": gpu, "amplicons_ms": {k: v[0] for k, v in out.items()}, "e2e_amplicons": e2e_line, "e2e": None,
    }
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
