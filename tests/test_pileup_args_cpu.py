"""`modkit pileup` / `pileup-hemi` argument checks without a GPU: every check that needs neither the device nor an input file
runs before the device is opened, so a bad command line gets its own error (exit 1, "> Error! <message>") on any machine and
leaves no output behind."""
import os
import subprocess

import pytest

from conftest import FIX, ROOT

MODKIT = os.path.join(ROOT, "modkit_b200", "_build", "modkit")
BAM = os.path.join(FIX, "bc_anchored_10_reads.sorted.bam")
DUPLEX = os.path.join(FIX, "duplex_modbam.sorted.bam")

# name: (subcommand, arguments before the inputs, output kind, message). "@REF" is a FASTA path that is never opened: these
# checks come before the FASTA is read.
ARG_ERRORS = {
    "percentile_above_one": ("pileup", ["-p", "1.5"], "bed", "filter percentile must be <= 1.0"),
    "hemi_needs_ref": ("pileup-hemi", ["--cpg"], "bed", "the following required arguments were not provided: --ref <REFERENCE_FASTA>"),
    "hemi_cpg_with_motif": ("pileup-hemi", ["--ref", "@REF", "--cpg", "--motif", "CG", "0"], "bed", "the argument '--cpg' cannot be used with '--motif <MOTIF> <MOTIF>'"),
    "hemi_needs_motif": ("pileup-hemi", ["--ref", "@REF"], "bed", "either --cpg or a --motif must be provided for pileup-hemi"),
    "hemi_motif_not_palindrome": ("pileup-hemi", ["--ref", "@REF", "--motif", "CA", "0"], "bed", "motif must be palindromic for pileup-hemi"),
    "partition_tag_length": ("pileup", ["--partition-tag", "HPX"], "dir", "illegal tag HPX should be length 2"),
    "partition_tag_repeated": ("pileup", ["--partition-tag", "HP", "--partition-tag", "HP"], "dir", "cannot repeat partition-tags, got HP twice"),
    "header_with_bedgraph": ("pileup", ["--bedgraph", "--header"], "dir", "the argument '--header' cannot be used with '--bedgraph' / '--partition-tag'"),
    "header_with_partition_tag": ("pileup", ["--partition-tag", "HP", "--header"], "dir", "the argument '--header' cannot be used with '--bedgraph' / '--partition-tag'"),
    "mixed_delim_with_bedgraph": ("pileup", ["--bedgraph", "--mixed-delim"], "dir", "the argument '--mixed-delim' cannot be used with '--bedgraph'"),
    "devices_with_bedgraph": ("pileup", ["--devices", "0,0", "--bedgraph"], "dir", "multi-GPU runs write one bedMethyl file through the device ingest"),
    "devices_with_host_ingest": ("pileup", ["--devices", "0,0", "--host-ingest"], "bed", "multi-GPU runs write one bedMethyl file through the device ingest"),
    "devices_to_stdout": ("pileup", ["--devices", "0,0"], "stdout", "multi-GPU runs need an output file (ranks write their slices at their offsets)"),
    "combine_strands_needs_motif": ("pileup", ["--combine-strands"], "bed", "need to specify either --motif or --cpg to combine strands"),
    "ignore_bad_code": ("pileup", ["--ignore", "mm"], "bed", "failed to parse mod code mm"),
    "edge_filter_not_a_number": ("pileup", ["--edge-filter", "x"], "bed", "stoul"),
    "preset_with_motif": ("pileup", ["--preset", "traditional", "--motif", "CG", "0"], "bed", "cannot use presets and motifs together"),
    "motif_repeated": ("pileup", ["--motif", "CG", "0", "--motif", "CG", "0"], "bed", "cannot have the same motif more than once"),
    "motif_bad_base": ("pileup", ["--motif", "CZ", "0"], "bed", "Invalid IUPAC code: Z"),
    "motif_offset_too_long": ("pileup", ["--motif", "CG", "5"], "bed", "motif not long enough for offset 5"),
    "motif_needs_ref": ("pileup", ["--cpg"], "bed", "reference fasta is required for using --motif or --cpg options"),
    # --preset traditional combines strands only after the "--motif or --cpg" check: it gets as far as the reference check
    "preset_needs_ref": ("pileup", ["--preset", "traditional"], "bed", "reference fasta is required for using --motif or --cpg options"),
    "combine_strands_not_palindrome": ("pileup", ["--combine-strands", "--ref", "@REF", "--motif", "CA", "0"], "bed", "cannot combine strands with a motif that is not a palindrome"),
}


def run(sub, args, bam, out):
    cmd = [MODKIT, sub] + args + [bam]
    if sub == "pileup":
        cmd.append(out)
    elif out != "-":
        cmd += ["-o", out]
    return subprocess.run(cmd, capture_output=True, text=True)


@pytest.mark.parametrize("case", sorted(ARG_ERRORS))
def test_argument_error_needs_no_device(case, native_lib, tmp_path):
    sub, args, kind, message = ARG_ERRORS[case]
    out = "-" if kind == "stdout" else str(tmp_path / ("out" if kind == "dir" else "out.bed"))
    args = [str(tmp_path / "ref.fa") if a == "@REF" else a for a in args]
    p = run(sub, args, DUPLEX if sub == "pileup-hemi" else BAM, out)
    assert p.returncode == 1 and p.stderr.startswith("> Error! " + message), p.stderr
    assert p.stdout == ""
    assert os.listdir(tmp_path) == []


def test_valid_command_line_reaches_the_device(native_lib, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    p = run("pileup", ["--no-filtering"], BAM, str(tmp_path / "out.bed"))
    assert p.returncode == 1 and p.stderr.startswith("> Error! no usable CUDA device"), p.stderr
    assert os.listdir(tmp_path) == []
