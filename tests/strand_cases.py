"""A truth set for `variants --vcf --strand` (test infrastructure): error-free full-span reads over a random reference
with alleles planted on chosen strands -- an SNV carried by forward reads only, a balanced SNV (as many forward as
reverse carriers, over a REF that is balanced too), an insertion carried by reverse reads only and a deletion carried
by forward reads only.  The strands come from synth.strands, with the carriers pinned to their strand."""
from __future__ import annotations

import numpy as np

from kindel_b200 import bamio, synth
from oracle import py_soracle as SO

OPS = "MIDNSHP=X"
L = 120
SNV_ONE, SNV_BAL, INS_AT, DEL_AT = 30, 60, 80, 95


def truth_set(seed=1):
    """(ref text, reads [(pos0, ops [(n, op)], seq, reverse)])."""
    rng = np.random.default_rng(seed)
    ref = "".join("ACGT"[i] for i in rng.integers(0, 4, L))

    def other(b):
        return "ACGT"[("ACGT".index(b) + 1) % 4]

    reads = []
    for k in range(54):
        seq = list(ref)
        ops = [(L, "M")]
        if k < 10:
            seq[SNV_ONE] = other(ref[SNV_ONE])
        elif k < 20:
            seq[SNV_BAL] = other(ref[SNV_BAL])
        elif k < 28:
            seq = seq[:INS_AT] + ["G", "T"] + seq[INS_AT:]
            ops = [(INS_AT, "M"), (2, "I"), (L - INS_AT, "M")]
        elif k < 36:
            seq = seq[:DEL_AT] + seq[DEL_AT + 2:]
            ops = [(DEL_AT, "M"), (2, "D"), (L - DEL_AT - 2, "M")]
        reads.append((0, ops, "".join(seq)))
    # forward: the one-strand SNV and deletion carriers, half the balanced SNV's, 4 plain reads; reverse: the rest --
    # 22 forward and 22 reverse REF reads at the balanced SNV
    fwd = list(range(0, 15)) + list(range(28, 36)) + list(range(36, 40))
    rev = list(range(15, 28)) + list(range(40, 54))
    strand = synth.strands(seed, len(reads), forward=fwd, reverse=rev)
    return ref, [r + (int(s),) for r, s in zip(reads, strand.tolist())]


def bam_records(reads, ref_id=0):
    return [(ref_id, p, 16 * rv, [(n << 4) | OPS.index(o) for n, o in ops], seq) for p, ops, seq, rv in reads]


def oracle_records(reads):
    return [SO.Rec(p + 1, seq, tuple(ops), rv) for p, ops, seq, rv in reads]


def write(tmp_path, seed=1):
    """(BAM path, FASTA path, ref text, reads) of the truth set."""
    ref, reads = truth_set(seed)
    bam, fa = tmp_path / ("strand%d.bam" % seed), tmp_path / ("strand%d.fa" % seed)
    bamio.write_bam(str(bam), [("t", L)], bam_records(reads))
    fa.write_text(">t\n" + ref + "\n")
    return bam, fa, ref, reads


def parse(lines):
    """{(POS, REF, ALT-field): (FILTER, INFO dict)}."""
    out = {}
    for ln in lines:
        f = ln.split("\t")
        info = dict(kv.split("=") if "=" in kv else (kv, True) for kv in f[7].split(";"))
        out[(int(f[1]), f[3], f[4])] = (f[6], info)
    return out


# ---- K8 results against bamio.select_reads, field for field ----------------------------------------------------
_ARRAYS = ("ref_start", "seq_off", "l_seq", "seq4", "contig_read_off", "complex_idx", "hard_idx")
_SCALARS = ("n_events", "reads_sorted", "max_simple_len", "reach_right", "reach_left")
_MASK = ("mask_read", "mask_off", "mask_qpos")


def fields(batch) -> dict:
    """The fields K8 produces, of a host ReadBatch (what select_reads gives)."""
    out = {f: np.asarray(getattr(batch, f)) for f in _ARRAYS}
    out.update({f: getattr(batch, f) for f in _SCALARS})
    out.update({f: (np.asarray(getattr(batch, f)) if batch.n_masked else None) for f in _MASK})
    return out


def assert_equal(got: dict, want: dict, what=""):
    for f in _ARRAYS:
        g, w = np.asarray(got[f]), np.asarray(want[f])
        assert g.shape == w.shape and np.array_equal(g.view(np.uint8) if g.size else g,
                                                     w.astype(g.dtype).view(np.uint8) if w.size else w.astype(g.dtype)), (what, f)
    for f in _SCALARS:
        assert int(got[f]) == int(want[f]), (what, f, got[f], want[f])
    for f in _MASK:
        if want[f] is None:
            assert got[f] is None, (what, f)
        else:
            assert got[f] is not None and np.array_equal(np.asarray(got[f], dtype=np.int64),
                                                         np.asarray(want[f], dtype=np.int64)), (what, f)
