"""Bench line of the base-quality QUAL (an extension, `variants --vcf --qual`): BASELINE.json configs[3]
(`cfg4_5Mb_200x`, as bench.py builds it) with the seeded qualities of synth.qualities.

    python tools/bench_variant_qual.py [--rounds R] [--out FILE]     # one JSON line on stdout (and in FILE)

Reports, on one GPU:
  * K11 (kdl_quality_pileup: K0 + K11 + K11g) against K0 + K1 (the pileup into a reused table), each the median of R
    alternating rounds timed with CUDA events, and K11's share of its floor: the bytes it must move -- seq4 and qual8
    read, qsum and emass written -- over the data sheet's 3.35 TB/s;
  * `parity`: the sha256 of qsum / emass against a restatement that never reads the engine (numpy per chunk of simple
    reads, oracle/py_qvoracle.py's walk for the complex ones);
  * the H2D time of qual8 from pinned memory;
  * on a 10^6-read BAM written with qualities, variants_vcf(qual=True) against variants_vcf(), wall clock, best of 3.
The card's name and power limit are read in the same run.  The default FILE is
profiles/h100_bench_n1_cfg4_5Mb_200x_qual.json."""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload generator and clock sampler of the main bench)

WORKLOAD = "cfg4_5Mb_200x"
HBM_TBPS = 3.35


def oracle_sums(batch, qual):
    """(qsum uint32 [4, n_slots], emass uint64 [n_slots]) without the engine: simple reads in numpy chunks (one M op at
    contig_slot + ref_start), complex reads through py_qvoracle.walk."""
    from oracle import py_oracle, py_qvoracle

    eps = np.array(py_qvoracle.EPS, dtype=np.int64)
    n_slots = int(batch.n_slots)
    qsum = np.zeros((4, n_slots), dtype=np.uint64)
    emass = np.zeros(n_slots, dtype=np.uint64)
    lens = batch.seq_len.astype(np.int64)
    qoff = np.concatenate(([0], np.cumsum(lens)))
    contig = np.repeat(np.arange(batch.n_contigs), np.diff(batch.contig_read_off))
    start = batch.contig_slot[contig].astype(np.int64) + batch.ref_start.astype(np.int64)
    simple = (batch.l_seq.astype(np.int64) & 0x80000000) == 0
    shifts = np.arange(28, -4, -4, dtype=np.uint32)
    step = 200_000
    for r0 in range(0, batch.n_reads, step):
        idx = np.flatnonzero(simple[r0:r0 + step]) + r0
        if idx.size == 0:
            continue
        ln = lens[idx]
        k = np.arange(int(ln.sum()), dtype=np.int64) - np.repeat(np.cumsum(ln) - ln, ln)
        rr = np.repeat(idx, ln)
        w = batch.seq4[batch.seq_off[rr].astype(np.int64) + (k >> 3)]
        nib = (w >> shifts[k & 7]) & 15
        q = qual[qoff[rr] + k].astype(np.uint64)
        slot = start[rr] + k
        for col, v in enumerate((1, 2, 4, 8)):
            m = nib == v
            qsum[col] += np.bincount(slot[m], weights=q[m], minlength=n_slots).astype(np.uint64)
        m = (nib == 1) | (nib == 2) | (nib == 4) | (nib == 8)
        # (float64 sums of integers below 2^53 are exact)
        emass += np.bincount(slot[m], weights=eps[np.minimum(q[m], 93).astype(np.int64)].astype(np.float64),
                             minlength=n_slots).astype(np.uint64)
    cx = np.flatnonzero(~simple)
    recs = py_oracle.records_of(batch)
    class Sparse(dict):  # a per-read accumulator that walk() can += into like a list
        def __missing__(self, key):
            return 0

    for r in cx.tolist():
        c = int(contig[r])
        L, s0 = int(batch.contig_len[c]), int(batch.contig_slot[c])
        q4, e = [Sparse() for _ in range(4)], Sparse()
        py_qvoracle.walk(L, recs[r], qual[qoff[r]:qoff[r + 1]].tolist(), set(), q4, e)
        for col in range(4):
            for p, v in q4[col].items():
                qsum[col, s0 + p] += np.uint64(v)
        for p, v in e.items():
            emass[s0 + p] += np.uint64(v)
    return qsum.astype(np.uint32), emass


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_n1_cfg4_5Mb_200x_qual.json"))
    ap.add_argument("--no-host", action="store_true", help="skip the end-to-end VCF timing")
    args = ap.parse_args(argv)

    import torch

    from kindel_b200 import _ffi, engine, synth
    from kindel_b200 import kindel as K

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _ffi.load()
    sampler = bench.ClockSampler(0)
    sampler.start()
    batch = bench.gen_reads(WORKLOAD)
    qual = synth.qualities(7, batch.seq_len)
    from kindel_b200 import bamio

    qual8 = bamio.qual_layout(batch, qual)
    n_slots = int(batch.n_slots)
    db = engine.upload(batch, dev)
    table = engine.CountTable(n_slots, dev)
    pinned = torch.from_numpy(qual8).pin_memory()
    q8 = pinned.to(dev)
    qsum = torch.empty((4, n_slots), dtype=torch.int32, device=dev)
    emass = torch.empty(n_slots, dtype=torch.int64, device=dev)
    stream = engine._stream_ptr(dev)

    def k11():
        _ffi.check(lib.kdl_quality_pileup(C.byref(db.struct), q8.data_ptr(), qsum.data_ptr(), emass.data_ptr(), n_slots,
                                          stream), "kdl_quality_pileup")

    def k1():
        engine.pileup(db, check=False, table=table)

    def timed(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        fn()
        ev[1].record()
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1])

    for _ in range(3):
        k11()
        k1()
    torch.cuda.synchronize()
    sampler.wait_first_sample()
    sampler.mark()
    t11, t1 = [], []
    for _ in range(args.rounds):
        t11.append(timed(k11))
        t1.append(timed(k1))
    h2d = []
    for _ in range(5):
        h2d.append(timed(lambda: q8.copy_(pinned, non_blocking=True)))
    clocks = sampler.stop()
    k11()
    torch.cuda.synchronize()
    got_q = qsum.cpu().numpy().view(np.uint32)
    got_e = emass.cpu().numpy().view(np.uint64)
    want_q, want_e = oracle_sums(batch, qual)
    sha = lambda a, b: hashlib.sha256(np.ascontiguousarray(a).tobytes() + np.ascontiguousarray(b).tobytes()).hexdigest()
    got, want = sha(got_q, got_e), sha(want_q, want_e)

    floor_bytes = 4 * int(batch.seq4.shape[0]) + qual8.nbytes + 24 * n_slots
    floor_ms = floor_bytes / (HBM_TBPS * 1e12) * 1e3
    k11_ms = statistics.median(t11)
    line = {
        "metric": "K11 quality sums (kdl_quality_pileup)", "data": "synthetic", "n_gpus": 1,
        "config": {"workload": WORKLOAD + "_qual", "reads": int(batch.n_reads), "complex_reads": int(batch.n_complex),
                   "hard_reads": int(batch.n_hard), "aligned_bases": int(batch.aligned_bases),
                   "tool": "tools/bench_variant_qual.py", "rounds": args.rounds},
        "parity": got == want, "sha256": got,
        "parity_oracle": "numpy over the simple reads + oracle/py_qvoracle.py's walk over the complex reads",
        "kernels_ms": {"k0_k11_k11g_median": k11_ms, "k0_k1_pileup": statistics.median(t1),
                       "k11_min": min(t11), "k11_max": max(t11)},
        "floor": {"bytes": floor_bytes, "hbm_tbps_datasheet": HBM_TBPS, "ms": floor_ms,
                  "share_of_floor": floor_ms / k11_ms},
        "h2d_qual8": {"bytes": int(qual8.nbytes), "ms_median": statistics.median(h2d),
                      "gb_per_s": qual8.nbytes / (statistics.median(h2d) * 1e-3) / 1e9},
        "clocks": clocks,
        "gpu": {"name": torch.cuda.get_device_name(dev), "count": 1,
                "power_limit_w": clocks.get("power_limit_w") if clocks else None},
    }
    del db, table, q8, qsum, emass, pinned
    torch.cuda.empty_cache()
    if not args.no_host:
        sub = synth.simple_reads(9, [5_000_000], 30)
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "q.bam")
            synth.write_simple_bam(path, sub, qual=synth.qualities(9, sub.seq_len))

            def best(**kw):
                ts = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    K.variants_vcf(path, **kw)
                    ts.append(time.perf_counter() - t0)
                return min(ts) * 1e3

            line["vcf_1e6_reads"] = {"reads": int(sub.n_reads), "ms_plain": best(), "ms_qual": best(qual=True),
                                     "ms_qual_min_qual_30": best(min_qual=30)}
    text = json.dumps(line)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text + "\n")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
