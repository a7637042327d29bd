"""-m gpu: the redundancy filter and the final .1aln order on the device's own raw records.  The raw
records of DeviceOverlaps.extend go through the product's fgb_filter and through the oracle's
orc_filter (oracle/fastga_oracle.c): same records, field by field and trace byte by trace byte, in the
same order.  The whole-path entry's final records, unsorted, give the reference's .1aln order
(aln_order_md5 of the recorded reference runs)."""
import os
import tempfile

import numpy as np
import pytest

import oracle_lib as ol
from fastga_b200 import formats, lib, synth

pytestmark = pytest.mark.gpu

#  name -> (make_pair arguments, contigs per scaffold) of the recorded e2e reference runs
PAIRS = {"small_pair": ((11, 1_200_000, 3, 0.05, 60_000), 1),
         "long_alignments": ((13, 6_000_000, 3, 0.03, 0), 1)}


def _pair(name):
    (seed, total, nc, div, sv), per = PAIRS[name]
    A, B = synth.make_pair(seed, total, nc, div, sv_every=sv)
    with tempfile.TemporaryDirectory() as wd:
        formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", per))
        formats.write_fasta(os.path.join(wd, "B.fasta"), synth.scaffolds_of(B, "sb", per))
        gA = formats.genome_from_fasta(os.path.join(wd, "A.fasta"))
        gB = formats.genome_from_fasta(os.path.join(wd, "B.fasta"))
    st = ol.reference("e2e/" + name, ol.digest(A, B, 8, per), None)
    return gA, gB, st


def _self_dup():
    import test_oracle_pin
    G = test_oracle_pin._self_genomes()["dup"]
    return formats.genome_from_arrays(G), ol.reference("self/dup", ol.digest(G), None)


def _device_raw(gA, gB):
    """the device's raw records (discovery order) and both filters on them"""
    self_mode = gB is None
    dA = lib.DeviceGenome(gA, want_revcomp=True)
    dB = dA if self_mode else lib.DeviceGenome(gB)
    xA = lib.DeviceGix.build(dA)
    amx = int(gA.clen.max())
    if self_mode:
        seeds = lib.DeviceSeeds.find_self(xA, amx, 10)
    else:
        xB = lib.DeviceGix.build(dB)
        seeds = lib.DeviceSeeds.find(xA, xB, amx, int(gB.clen.max()), 10)
        xB.close()
    xA.close()
    jb, ib = seeds.layout[2], seeds.layout[3]
    ov = lib.DeviceOverlaps.extend(seeds, dA, dB, gA.freq)
    recs, buf = ov.records()
    product = lib.filter_overlaps(ov.h, dA.perm, dB.perm, jb, ib)
    perm1, perm2 = dA.perm.copy(), dB.perm.copy()
    ov.close()
    seeds.close()
    dA.close()
    if not self_mode:
        dB.close()
    return recs, buf, product, perm1, perm2, jb, ib


def _oracle_filter(recs, buf, perm1, perm2, jb, ib):
    """orc_filter on the device's raw records.  The discovery order holds each align_contigs call's
    records together, so a call is a run of one (strand, contig pair) in that order."""
    pk = recs["pairkey"].astype(np.int64)
    ov = np.zeros(len(recs), dtype=ol.OVL_DT)
    ov["comp"] = pk >> (jb + ib)
    ov["aread"] = perm1[(pk >> jb) & ((1 << ib) - 1)]
    ov["bread"] = perm2[pk & ((1 << jb) - 1)]
    for f in ("abpos", "bbpos", "aepos", "bepos", "diffs", "tlen"):
        ov[f] = recs[f]
    ov["grp"] = np.concatenate([[0], np.cumsum(pk[1:] != pk[:-1])]) if len(pk) else []
    ov["toff"] = recs["toff"]
    al = ol.filter(ov, buf)
    return al, ol.filter_counters()


@pytest.mark.parametrize("name", ["small_pair", "long_alignments", "self_dup"])
def test_device_raw_records_filter_like_the_oracle(name):
    if name == "self_dup":
        gA, st = _self_dup()
        gB, fastga = None, (lambda: lib.fastga_self(gA))
    else:
        gA, gB, st = _pair(name)
        fastga = (lambda: lib.fastga(gA, gB))
    recs, buf, product, perm1, perm2, jb, ib = _device_raw(gA, gB)
    assert len(recs) == st["alns"]
    want, cnt = _oracle_filter(recs, buf, perm1, perm2, jb, ib)
    print(name, "raw", len(recs), "kept", len(want), {k: v for k, v in cnt.items() if v})
    assert ol.alignment_differences(product, want) == ""
    assert len(want) == st["records"]
    assert ol.md5_lines(want.canonical_lines_unsorted()) == st["aln_order_md5"]
    alns, _ = fastga()
    assert ol.md5_lines(alns.canonical_lines_unsorted()) == st["aln_order_md5"]
