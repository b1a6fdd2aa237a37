"""`kindel` command line on the H100 engine (restates the argh CLI of reference kindel/cli.py:9-66).

Sub-commands, flags, defaults and output streams follow the reference: `consensus` prints the
REPORT blocks to stderr and one `>name` / sequence pair per contig to stdout (cli.py:30-33; with the `--fastq`
extension one FASTQ record per contig instead),
`weights` / `features` write TSV to stdout (cli.py:44,50), `version` prints `kindel <version>`;
`variants` (in the reference's README only) is an extension, see kindel.variants; its `--vcf` writes a sites-only VCF
(kindel.variants_vcf), against a FASTA with `--reference`, with per-strand counts and a strand odds ratio with
`--strand` / `--max-sor`, with a base-quality QUAL with `--qual` / `--min-qual`, with its indels left-aligned with
`--left-align`.  `--primers scheme.bed` (consensus, weights, features, variants) masks the amplicon primer
bases of every read before the pileup (kindel_b200/primers.py); `--mask-overlaps` counts each read pair once where
its mates overlap (include/kindel_b200.h K10); `--normalise N` with a named scheme keeps at most N reads of each
amplicon and strand (K12 + K13, include/kindel_b200.h); `--dedup` removes duplicate reads and read pairs (K14).  `amplicons --primers scheme.bed` (an extension) writes a TSV row per
sample and amplicon of a tiled scheme: its reads (K12) and the depth of its insert (K12d).
argh derived the flags from the function signatures (first letter as short option unless two
parameters share it); argparse spells the same set out.  Note the CLI default `--min-overlap 7`
(cli.py:13) differs from the API default 9 (kindel.py:492), as in the reference.
"""
from __future__ import annotations

import argparse
import sys

from . import __version__


def consensus(bam_path, realign=False, min_depth=1, min_overlap=7, clip_decay_threshold=0.1, mask_ends=50,
              trim_ends=False, uppercase=False, gpus=None, iupac_threshold=None, fastq=False, quality_vote=False,
              **filters):
    """Infer consensus sequence(s) from alignment in SAM/BAM format"""
    from . import kindel

    res = kindel.bam_to_consensus(bam_path, realign, min_depth, min_overlap, clip_decay_threshold, mask_ends,
                                  trim_ends, uppercase, devices=gpus, iupac_threshold=iupac_threshold,
                                  qualities=fastq, quality_vote=quality_vote, **filters)
    print("\n".join(res.refs_reports.values()), file=sys.stderr)
    for record in res.consensuses:
        if fastq:  # extension: @name, sequence, +, Phred+33 qualities
            print(f"@{record.name}\n{record.sequence}\n+\n{record.qualities}")
        else:
            print(f">{record.name}")
            print(record.sequence)


def weights(bam_path, relative=False, confidence=True, confidence_alpha=0.01, gpus=None, **filters):
    """Returns table of per-site nucleotide frequencies and coverage"""
    from . import kindel

    kindel.weights(bam_path, relative, confidence, confidence_alpha, devices=gpus, **filters).to_csv(
        sys.stdout, sep="\t", index=False)


def features(bam_path, gpus=None, **filters):
    """Returns table of per-site nucleotide frequencies and coverage including indels"""
    from . import kindel

    kindel.features(bam_path, devices=gpus, **filters).to_csv(sys.stdout, sep="\t", index=False)


def variants(bam_path, abs_threshold=1, rel_threshold=0.01, only_variants=False, absolute=False, gpus=None, vcf=False,
             reference=None, strand=False, max_sor=None, qual=False, min_qual=None, left_align=False, **filters):
    """Output variants exceeding specified absolute and relative frequency thresholds"""
    from . import kindel

    if vcf:  # extension: the sites of --only-variants as a sites-only VCF (against --reference when given)
        extra = {} if reference is None else dict(reference=reference)
        if strand or max_sor is not None:  # extension: ADF / ADR / SOR (and FILTER sor)
            extra.update(strand=True, max_sor=max_sor)
        if qual or min_qual is not None:  # extension: QUAL, BQ / AQ (and FILTER lowqual)
            extra.update(qual=True, min_qual=min_qual)
        if left_align:  # extension: indels moved to their leftmost place against the reference
            extra.update(left_align=True)
        sys.stdout.write(kindel.variants_vcf(bam_path, abs_threshold, rel_threshold, devices=gpus, **filters, **extra))
        return
    kindel.variants(bam_path, abs_threshold, rel_threshold, only_variants, absolute, devices=gpus, **filters).to_csv(
        sys.stdout, sep="\t", index=False)


def amplicons(bam_paths, primers, min_depth=20, gpus=None, **filters):
    """Report each amplicon's reads and insert depth per sample (tiled amplicon schemes)"""
    from . import kindel

    df = kindel.amplicons(bam_paths, primers, min_depth, devices=gpus, **filters)
    capped = df.attrs.get("dropped", {})  # (--normalise)
    duplicates = df.attrs.get("duplicates", {})  # (--dedup)
    for name, (kept, assigned, unprimed, mispaired, ambiguous) in df.attrs["reads"].items():
        rows = df[df["sample"] == name]
        drop = rows.loc[rows["status"] == "dropout", "amplicon"].tolist()
        print("%s: %d reads kept: %d assigned, %d unprimed, %d mispaired, %d ambiguous; %d amplicons, %d dropouts%s%s%s"
              % (name, kept, assigned, unprimed, mispaired, ambiguous, len(rows), len(drop),
                 (": " + ", ".join(drop)) if drop else "",
                 "; %d reads over the normalise cap dropped" % capped[name] if name in capped else "",
                 "; %d duplicate reads removed" % duplicates[name] if name in duplicates else ""),
              file=sys.stderr)
    out = ["\t".join(kindel.AMPLICON_COLUMNS)]
    for r in df.itertuples(index=False):
        out.append("%s\t%s\t%s\t%s\t%d\t%d\t%d\t%d\t%d\t%.2f\t%d\t%.4f\t%s"
                   % (r.sample, r.contig, r.amplicon, r.pool, r.start, r.end, r.insert_start, r.insert_end, r.reads,
                      r.mean_depth, r.lowest_depth, r.covered, r.status))
    sys.stdout.write("\n".join(out) + "\n")


def plot(bam_path):
    """Plot sitewise soft clipping frequency across reference and genome"""
    from . import kindel

    return kindel.plotly_clips(bam_path)


def version():
    """Show version"""
    return f"kindel {__version__}"


def _add_gpus(p):
    # extension (not in the reference's CLI): shard the pileup over the GPUs of this node
    p.add_argument("--gpus", type=int, default=None,
                   help="number of GPUs of this node to shard the pileup over (default: $KINDEL_GPUS or 1)")


def _flags(text: str) -> int:
    return int(text, 0)  # decimal or 0x...


def _add_filters(p):
    # extension (not in the reference's CLI): read and base filters, all off by default
    p.add_argument("--min-base-quality", type=int, default=0,
                   help="mask bases with Phred quality below this value (read as N, not counted)")
    p.add_argument("--min-mapq", type=int, default=0, help="skip records with mapping quality below this value")
    p.add_argument("--exclude-flags", type=_flags, default=0,
                   help="skip records with any of these FLAG bits set (decimal or 0x...)")
    # extension: amplicon primer masking, off by default
    p.add_argument("--primers", default=None, metavar="BED",
                   help="mask the bases of each read that lie in an amplicon primer of this BED (plain or gzip): read "
                        "as N, not counted")
    # extension: each read pair counted once where its mates overlap, off by default
    p.add_argument("--mask-overlaps", action="store_true",
                   help="count each read pair once where its mates overlap: the second mate's bases, deletions and "
                        "insertions there are not counted where the first mate has information")
    # extension: depth normalisation of amplicon data, off by default
    p.add_argument("--normalise", type=_normalise, default=None, metavar="N",
                   help="keep only the first N reads (file order) of each amplicon and strand of the --primers "
                        "scheme, whose 4th column names each primer <amplicon>_LEFT or <amplicon>_RIGHT")
    # extension: duplicate removal, off by default
    p.add_argument("--dedup", action="store_true",
                   help="remove duplicate reads and read pairs (same unclipped 5' ends and strands) before the "
                        "pileup, keeping the one with the highest sum of base qualities >= 15, as samtools markdup -r")


def _normalise(text: str) -> int:
    from .kindel import check_normalise

    return check_normalise(int(text))  # ValueError (not an integer, below 1) -> argparse error


def _iupac_threshold(text: str) -> float:
    from .kindel import check_iupac_threshold

    return check_iupac_threshold(float(text))  # ValueError (NaN, outside [0, 1]) -> argparse error


def _max_sor(text: str) -> float:
    from .vcf import check_number

    return check_number(float(text), "max_sor")  # ValueError (NaN) -> argparse error


def _min_qual(text: str) -> float:
    from .vcf import check_number

    return check_number(float(text), "min_qual")  # ValueError (NaN) -> argparse error


def _filters(a) -> dict:
    out = dict(min_base_quality=a.min_base_quality, min_mapq=a.min_mapq, exclude_flags=a.exclude_flags)
    if a.primers is not None:  # (the keyword only when given: every call without it stays as it was)
        out["primers"] = a.primers
    if a.mask_overlaps:
        out["mask_overlaps"] = True
    if a.normalise is not None:
        out["normalise"] = a.normalise
    if a.dedup:
        out["dedup"] = True
    return out


def _amplicon_filters(a) -> dict:
    out = _filters(a)
    del out["primers"]  # (the scheme itself)
    return out


def build_parser() -> argparse.ArgumentParser:
    fmt = argparse.ArgumentDefaultsHelpFormatter
    parser = argparse.ArgumentParser(prog="kindel", formatter_class=fmt)
    sub = parser.add_subparsers(dest="command")

    p = sub.add_parser("consensus", help=consensus.__doc__, description=consensus.__doc__, formatter_class=fmt)
    p.add_argument("bam_path", help="path to SAM/BAM file")
    p.add_argument("-r", "--realign", action="store_true",
                   help="attempt to reconstruct reference around soft-clip boundaries")
    p.add_argument("--min-depth", type=int, default=1, help="substitute Ns at coverage depths beneath this value")
    p.add_argument("--min-overlap", type=int, default=7, help="match length required to close soft-clipped gaps")
    p.add_argument("-c", "--clip-decay-threshold", type=float, default=0.1,
                   help="read depth fraction at which to cease clip extension")
    p.add_argument("--mask-ends", type=int, default=50,
                   help="ignore clip dominant positions within n positions of termini")
    p.add_argument("-t", "--trim-ends", action="store_true",
                   help="trim ambiguous nucleotides (Ns) from sequence ends")
    p.add_argument("-u", "--uppercase", action="store_true", help="close gaps using uppercase alphabet")
    _add_gpus(p)
    _add_filters(p)
    # extension (not in the reference's CLI): IUPAC ambiguity codes for mixed sites, off by default
    p.add_argument("--iupac-threshold", type=_iupac_threshold, default=None, metavar="F",
                   help="emit the IUPAC code of the fewest most frequent bases that reach this fraction (0-1) of "
                        "the depth instead of the majority base")
    # extension (not in the reference's CLI): per-base qualities, off by default
    p.add_argument("--fastq", action="store_true",
                   help="write FASTQ with a Phred quality per consensus base instead of FASTA")
    # extension (not in the reference's CLI): the base by the reads' base qualities, off by default
    p.add_argument("--quality-vote", action="store_true",
                   help="emit the base whose reads' base qualities give it the largest summed log-likelihood weight "
                        "instead of the majority base (not with --iupac-threshold)")
    p.set_defaults(func=lambda a: consensus(a.bam_path, a.realign, a.min_depth, a.min_overlap,
                                            a.clip_decay_threshold, a.mask_ends, a.trim_ends, a.uppercase, a.gpus,
                                            a.iupac_threshold, a.fastq, a.quality_vote, **_filters(a)))

    p = sub.add_parser("weights", help=weights.__doc__, description=weights.__doc__, formatter_class=fmt)
    p.add_argument("bam_path", help="path to SAM/BAM file")
    p.add_argument("-r", "--relative", action="store_true", help="output relative nucleotide frequencies")
    p.add_argument("-c", "--confidence", action="store_false", default=True,
                   help="calculate confidence interval for consensus")
    p.add_argument("--confidence-alpha", type=float, default=0.01, help="confidence interval alpha value")
    _add_gpus(p)
    _add_filters(p)
    p.set_defaults(func=lambda a: weights(a.bam_path, a.relative, a.confidence, a.confidence_alpha, a.gpus,
                                          **_filters(a)))

    p = sub.add_parser("features", help=features.__doc__, description=features.__doc__, formatter_class=fmt)
    p.add_argument("bam_path", help="path to SAM/BAM file")
    _add_gpus(p)
    _add_filters(p)
    p.set_defaults(func=lambda a: features(a.bam_path, a.gpus, **_filters(a)))

    # `variants` is listed by the reference's README (README.md:106-107) but absent from its code: an extension here
    p = sub.add_parser("variants", help=variants.__doc__, description=variants.__doc__, formatter_class=fmt)
    # extension: several files (with --vcf) give one VCF with a column per sample
    p.add_argument("bam_path", nargs="+",
                   help="path to SAM/BAM file; with --vcf several files give one VCF with a column per sample")
    p.add_argument("-a", "--abs-threshold", type=int, default=1, help="absolute frequency above which to call variants")
    p.add_argument("-r", "--rel-threshold", type=float, default=0.01,
                   help="relative frequency (0.0-1.0) above which to call variants")
    p.add_argument("-o", "--only-variants", action="store_true", help="exclude invariant sites from output")
    p.add_argument("--absolute", action="store_true", help="report absolute variant frequencies")
    _add_gpus(p)
    _add_filters(p)
    # extension: the variant sites as VCF (REF = the sample's most frequent allele; see kindel.variants_vcf)
    p.add_argument("--vcf", action="store_true",
                   help="write the variant sites as a sites-only VCF 4.2 instead of the table")
    # extension: REF from the FASTA the alignment was made against; SNVs, insertions and deletions against it (no
    # short option: -r is --rel-threshold)
    p.add_argument("--reference", default=None, metavar="FASTA",
                   help="with --vcf: call SNVs, insertions and deletions against this FASTA (plain or gzip)")
    # extension: forward / reverse strand counts and the strand odds ratio of every record, and a filter on it
    p.add_argument("--strand", action="store_true",
                   help="with --vcf: add ADF / ADR (per-strand allele counts) and SOR (strand odds ratio) to INFO")
    p.add_argument("--max-sor", type=_max_sor, default=None, metavar="X",
                   help="with --vcf: FILTER `sor` where an ALT's strand odds ratio is above X (implies --strand)")
    # extension: a QUAL from the reads' base qualities, the per-allele qualities in INFO, and a filter on it
    p.add_argument("--qual", action="store_true",
                   help="with --vcf: QUAL from the base qualities (Poisson error model), BQ / AQ in INFO")
    p.add_argument("--min-qual", type=_min_qual, default=None, metavar="X",
                   help="with --vcf: FILTER `lowqual` where QUAL is below X (implies --qual)")
    # extension: every indel moved to its leftmost place against the reference before the events are counted
    p.add_argument("--left-align", action="store_true",
                   help="with --vcf --reference: left-align insertions and deletions against the reference before they "
                        "are grouped and counted")
    p.set_defaults(func=lambda a: variants(a.bam_path[0] if len(a.bam_path) == 1 else a.bam_path, a.abs_threshold,
                                           a.rel_threshold, a.only_variants, a.absolute, a.gpus, a.vcf, a.reference,
                                           a.strand, a.max_sor, a.qual, a.min_qual, a.left_align, **_filters(a)))

    # extension: per-amplicon reads and depth of a tiled primer scheme (the BED's name column says which primers pair)
    p = sub.add_parser("amplicons", help=amplicons.__doc__, description=amplicons.__doc__, formatter_class=fmt)
    p.add_argument("bam_path", nargs="+", help="path to SAM/BAM file; several files give one row block per sample")
    p.add_argument("--min-depth", type=int, default=20,
                   help="an amplicon whose insert's mean depth is below this is a dropout; `covered` counts its "
                        "positions at or above it")
    _add_gpus(p)
    _add_filters(p)
    p.set_defaults(func=lambda a: amplicons(a.bam_path, a.primers, a.min_depth, a.gpus, **_amplicon_filters(a)))

    p = sub.add_parser("plot", help=plot.__doc__, description=plot.__doc__, formatter_class=fmt)
    p.add_argument("bam_path", help="path to SAM/BAM file")
    p.set_defaults(func=lambda a: plot(a.bam_path))

    p = sub.add_parser("version", help=version.__doc__, description=version.__doc__)
    p.set_defaults(func=lambda a: version())
    return parser


def _check_consensus_args(parser, args):
    if getattr(args, "command", None) == "consensus" and args.quality_vote and args.iupac_threshold is not None:
        parser.error("consensus: --quality-vote cannot be combined with --iupac-threshold")


def _check_variants_args(parser, args):
    # --absolute and --only-variants shape the table; the VCF always holds the variant sites alone
    paths = getattr(args, "bam_path", None)
    if getattr(args, "command", None) == "variants" and len(paths) > 1:
        if not args.vcf:
            parser.error("variants: several alignment files need --vcf (the table has no sample columns)")
        if args.strand or args.max_sor is not None:
            parser.error("variants: --strand and --max-sor take one alignment file")
        if args.qual or args.min_qual is not None:
            parser.error("variants: --qual and --min-qual take one alignment file")
    if getattr(args, "left_align", False) and (not args.vcf or args.reference is None):
        parser.error("variants: --left-align needs --vcf and --reference (the indels move against its bases)")
    if getattr(args, "vcf", False):
        for flag, on in (("--absolute", args.absolute), ("--only-variants", args.only_variants)):
            if on:
                parser.error("variants: --vcf cannot be combined with %s (a table option)" % flag)
    elif getattr(args, "reference", None) is not None:
        parser.error("variants: --reference needs --vcf (the table has no reference mode)")
    elif getattr(args, "strand", False) or getattr(args, "max_sor", None) is not None:
        parser.error("variants: --strand and --max-sor need --vcf (the table has no strand columns)")
    elif getattr(args, "qual", False) or getattr(args, "min_qual", None) is not None:
        parser.error("variants: --qual and --min-qual need --vcf (the table has no QUAL)")


def _check_normalise_args(parser, args):
    if getattr(args, "normalise", None) is None:
        return
    if args.primers is None:
        parser.error("--normalise needs --primers (a primer BED whose 4th column names each primer <amplicon>_LEFT "
                     "or <amplicon>_RIGHT)")
    from .primers import load_scheme

    try:
        load_scheme(args.primers)
    except (OSError, ValueError) as e:
        parser.error("--normalise needs a named primer scheme: %s" % e)


def _check_amplicons_args(parser, args):
    if getattr(args, "command", None) == "amplicons" and args.primers is None:
        parser.error("amplicons: --primers is required (a primer BED whose 4th column names each primer "
                     "<amplicon>_LEFT or <amplicon>_RIGHT)")


def main(argv=None):
    parser = build_parser()
    args = parser.parse_args(argv)
    _check_amplicons_args(parser, args)
    _check_normalise_args(parser, args)
    _check_consensus_args(parser, args)
    _check_variants_args(parser, args)
    if not getattr(args, "func", None):
        parser.print_usage()
        return 1
    out = args.func(args)
    if out is not None:  # argh prints a command's return value
        print(out)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
