"""-m gpu: the whole-path calls (fgb_fastga, fgb_fastga_self) report the counts the stage calls give on the
same input, in pair and in SELF mode."""
import pytest

import self_cases as sc
from fastga_b200 import formats, lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", ["pair", "self"])
def test_whole_path_stats_match_the_stage_calls(mode, small_pair):
    self_mode = mode == "self"
    if self_mode:
        gA = gB = formats.genome_from_arrays(sc.straddle_genome())
        _, stats = lib.fastga_self(gA)
    else:
        gA, gB = small_pair
        _, stats = lib.fastga(gA, gB)
    dA = lib.DeviceGenome(gA, want_revcomp=True)
    dB = dA if self_mode else lib.DeviceGenome(gB)
    xA = lib.DeviceGix.build(dA)
    xB = xA if self_mode else lib.DeviceGix.build(dB)
    amx, bmx = int(gA.clen.max()), int(gB.clen.max())
    assert (stats["nkmers1"], stats["nkmers2"]) == (xA.n, xB.n)
    # the entries of table 1 the merge reads: its forward strand, or in SELF mode all of it
    assert stats["nkmers1_fwd"] == (xA.n if self_mode else lib.DeviceGix.build_forward(dA).n)
    S = lib.DeviceSeeds.find_self(xA, amx) if self_mode else lib.DeviceSeeds.find(xA, xB, amx, bmx)
    xA.close()
    xB.close()
    assert (stats["nseeds"], stats["sumlen"]) == (S.n, S.sumlen)
    cnt = lib.DeviceOverlaps.extend(S, dA, dB, gA.freq).counters()
    for k, c in (("nhits", "hits"), ("nla", "la_calls"), ("nwaves", "waves"), ("ncells", "cells"),
                 ("nseg", "nseg"), ("nwork", "nwork")):
        assert stats[k] == cnt[c], k
