"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/reference_digests.json from the UNMODIFIED reference.

Needs the reference tree (oracle/refload.py finds it):   python -m oracle.make_reference_digests

The differential tests that compared the C oracle and the host half of the API with the reference itself
(tests/test_fuzz_parity.py, tests/test_fuzz_host_api.py, tests/test_oracle_pin.py) compare with this file instead,
so they need nothing outside the repository.  It holds, as truncated sha256 digests of canonical JSON:
  fuzz_pileup   per fuzz case (tests/fuzz_cases.py): the exception `parse_bam` raises, or per contig its table
                (tests/helpers.reference_alignment_to_table), insertion dicts and `changes`
  host_api      per clip-heavy / generic case and its option set (`options`): what `bam_to_consensus` returns
                or raises, the CDR helpers on every contig, and the `weights` / `features` frames
  suite_fasta   the FASTA files of the reference's own test suite, per fixture and mode (plain / realign)
  limit_cases   per group of tests/limit_cases.py: per contig its table, insertion dicts and `changes`, and the
                FASTA of `bam_to_consensus` with the default options

`python -m oracle.make_reference_digests limit_cases` recomputes only the named sections of an existing file.
"""
from __future__ import annotations

import glob
import hashlib
import json
import os
import random
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

OUT = os.path.join(ROOT, "tests", "golden", "reference_digests.json")
N_FUZZ = 400      # tests/test_fuzz_parity.py
N_CLIP = 160      # tests/test_fuzz_host_api.py
N_GENERIC = 400
FRAME_EVERY = {"clip": 4, "gen": 3}  # the frames of every 4th clip case / 3rd generic case
SUITE_DIRS = ("data_bwa_mem", "data_minimap2", "data_ext")


def digest(obj) -> str:
    return hashlib.sha256(json.dumps(obj, separators=(",", ":")).encode()).hexdigest()[:12]


def options(seed):
    """The option set of host-API case `seed` (bam_to_consensus keywords)."""
    rng = random.Random(seed)
    return dict(realign=rng.random() < 0.8, min_depth=rng.choice([1, 1, 2, 5]), min_overlap=rng.choice([1, 3, 7, 9]),
                clip_decay_threshold=rng.choice([0.0, 0.1, 0.1, 0.3, 0.9]), mask_ends=rng.choice([0, 1, 5, 20, 50]),
                trim_ends=rng.random() < 0.5, uppercase=rng.random() < 0.3)


def option_args(o):
    return (o["realign"], o["min_depth"], o["min_overlap"], o["clip_decay_threshold"], o["mask_ends"], o["trim_ends"],
            o["uppercase"])


def frame_options(seed):
    rng = random.Random(seed)
    return rng.random() < 0.5, rng.random() < 0.7, rng.choice([0.01, 0.05, 0.2])


def table_digest(table, ins, changes):
    """One contig of a pileup: table [19, L+1], insertion dicts of slots 0..L (OrderedDicts), changes list."""
    return {"table": digest([[int(x) for x in row] for row in table]),
            "ins": digest([[i, list(d.items())] for i, d in enumerate(ins) if d]),
            "changes": digest(list(changes))}


def result_digest(res, path):
    return {"consensus": digest([[r.name, r.sequence] for r in res.consensuses]),
            "changes": digest([[c, list(ch)] for c, ch in res.refs_changes.items()]),
            "reports": digest([[c, rep.replace(str(path), "<bam>")] for c, rep in res.refs_reports.items()])}


def regions(rs):
    return [list(r) for r in rs]


def cdr_digest(k, args_f, args_r, args_p, min_overlap):
    """cdr_start / cdr_end / cdrp / merge_cdrps of one contig, through module `k` (reference or port)."""
    pairs = k.cdrp_consensuses(*args_p)
    return digest([regions(k.cdr_start_consensuses(*args_f)), regions(k.cdr_end_consensuses(*args_r)),
                   [[list(f), list(r)] for f, r in pairs], regions(k.merge_cdrps(pairs, min_overlap))])


def cdr_args(aln, o):
    """The arguments the reference's tests pass to the CDR helpers, from an `alignment`-shaped record."""
    t, m = o["clip_decay_threshold"], o["mask_ends"]
    return ((aln.weights, aln.deletions, aln.clip_start_weights, aln.clip_start_depth, t, m),
            (aln.weights, aln.deletions, aln.clip_end_weights, aln.clip_end_depth, t, m),
            (aln.weights, aln.deletions, aln.clip_start_weights, aln.clip_end_weights, aln.clip_start_depth,
             aln.clip_end_depth, t, m))


def frame_digest(df):
    return digest([df.to_csv(), [str(t) for t in df.dtypes], [str(c) for c in df.columns], type(df.index).__name__,
                   str(df.index.dtype)])


def fasta_digest(records):
    return digest(sorted([name, seq] for name, seq in records))


def _fuzz_pileup(k, tmp):
    from fuzz_cases import random_case

    out = []
    for seed in range(N_FUZZ):
        path = os.path.join(tmp, "fuzz%d.sam" % seed)
        with open(path, "w") as fh:
            fh.write(random_case(seed))
        out.append(_fuzz_pileup_one(k, path))
    return out


def _fuzz_pileup_one(k, path):
    import helpers

    try:
        alns = k.parse_bam(path)
    except IndexError:
        return {"raises": ["IndexError"]}
    except KeyError as exc:
        return {"raises": ["KeyError", exc.args[0]]}
    contigs = []
    for aln in alns.values():
        t, ins = helpers.reference_alignment_to_table(aln)
        _, changes = k.consensus_sequence(aln.weights, aln.insertions, aln.deletions, None, False, 1, False)
        contigs.append(table_digest(t, ins, changes))
    return {"raises": None, "contigs": list(alns), "digests": contigs}


def _host_api(k, tmp, kind):
    from clip_cases import clip_case
    from fuzz_cases import random_case

    make, n = (clip_case, N_CLIP) if kind == "clip" else (random_case, N_GENERIC)
    out = []
    for seed in range(n):
        path = os.path.join(tmp, "%s%d.sam" % (kind, seed))
        with open(path, "w") as fh:
            fh.write(make(seed))
        o = options(seed)
        try:
            res = k.bam_to_consensus(path, *option_args(o))
        except (IndexError, KeyError) as exc:
            out.append({"raises": type(exc).__name__})
            continue
        entry = {"raises": None, **result_digest(res, path)}
        entry["cdr"] = [cdr_digest(k, *cdr_args(aln, o), o["min_overlap"]) for aln in k.parse_bam(path).values()]
        if seed % FRAME_EVERY[kind] == 0:
            entry["weights"] = frame_digest(k.weights(path, *frame_options(seed)))
            try:
                entry["features"] = frame_digest(k.features(path))
            except IndexError:
                entry["features"] = "IndexError"
        out.append(entry)
    return out


def _limit_cases(k, tmp):
    import limit_cases

    out = {}
    for name in limit_cases.GROUPS:
        path = os.path.join(tmp, name + ".sam")
        with open(path, "w") as fh:
            fh.write(limit_cases.sam_text(name))
        entry = _fuzz_pileup_one(k, path)
        res = k.bam_to_consensus(path)
        entry["fasta"] = fasta_digest([(r.name, r.sequence) for r in res.consensuses])
        out[name] = entry
    return out


def _suite_fasta(root):
    def fasta(path):
        recs, name = {}, None
        for line in open(path):
            line = line.strip()
            if line.startswith(">"):
                name = line[1:]
                recs[name] = ""
            elif name:
                recs[name] += line
        return recs

    out = {}
    for d in SUITE_DIRS:
        for p in sorted(glob.glob(os.path.join(root, "tests", d, "*.bam")) + glob.glob(os.path.join(root, "tests", d, "*.sam"))):
            for suf in (".fa", ".realign.fa"):
                fa = os.path.splitext(p)[0] + suf
                if os.path.isfile(fa):
                    out["tests/%s/%s%s" % (d, os.path.basename(p), suf)] = fasta_digest(fasta(fa).items())
    return out


def main():
    from oracle import refload

    if not refload.available() or not os.path.isdir(os.path.join(refload.REFERENCE_ROOT, "tests")):
        raise SystemExit("the reference tree (with its tests/) is not present")
    k = refload.load_reference()
    sections = {"fuzz_pileup": lambda tmp: _fuzz_pileup(k, tmp),
                "host_api": lambda tmp: {"clip": _host_api(k, tmp, "clip"), "gen": _host_api(k, tmp, "gen")},
                "suite_fasta": lambda tmp: _suite_fasta(refload.REFERENCE_ROOT),
                "limit_cases": lambda tmp: _limit_cases(k, tmp)}
    only = sys.argv[1:]
    if any(s not in sections for s in only):
        raise SystemExit("sections: " + ", ".join(sections))
    doc = {"reference": "bede/kindel v1.2.1 @ 14d727b", "generator": "oracle/make_reference_digests.py"}
    if only:
        with open(OUT) as fh:
            doc = json.load(fh)
    with tempfile.TemporaryDirectory() as tmp:
        for name, make in sections.items():
            if not only or name in only:
                doc[name] = make(tmp)
    with open(OUT, "w") as fh:
        json.dump(doc, fh, separators=(",", ":"), sort_keys=True)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
