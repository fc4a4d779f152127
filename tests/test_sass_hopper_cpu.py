"""SASS evidence (no GPU needed): the kernels DESIGN.md §4 describes as wgmma / TMA kernels really contain the Hopper
instructions — HGMMA (wgmma.mma_async), WARPGROUP.ARRIVE / DEPBAR (wgmma.fence / wait_group), UTMALDG
(cp.async.bulk.tensor, .MULTICAST for the CTA pair), SYNCS (mbarrier) — and the programmatic-launch pair PREEXIT / ACQBULK
(griddepcontrol.launch_dependents / .wait)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXPECT = {
    # object -> {mnemonic regex: minimum occurrences}
    "gemm_tc.o": {r"HGMMA\.64x256x16\.F32\.BF16": 50, r"HGMMA\.64x16x16\.F32\.BF16": 50, r"UTMALDG\.2D\b": 100,
                  r"UTMAPF\.L2\.2D": 10, r"WARPGROUP\.DEPBAR": 10, r"SYNCS\.PHASECHK": 10, "ACQBULK": 10, "PREEXIT": 10},
    "gemm_tc2.o": {r"HGMMA\.64x256x16\.F32\.BF16": 50, r"UTMALDG\.2D\.MULTICAST": 20, r"SYNCS\.ARRIVE\.TRANS64\.RED": 10,
                   r"UCGABAR_(ARV|WAIT)": 4, "ACQBULK": 4},
    "attention_tc.o": {r"HGMMA\.64x128x16\.F32\.BF16": 16, r"UTMALDG\.5D": 8, r"WARPGROUP\.DEPBAR": 2, "ACQBULK": 1},
    "gemv_ks.o": {"ACQBULK": 50, "PREEXIT": 50},
    "attention.o": {"ACQBULK": 2, r"UCGABAR_(ARV|WAIT)": 2},   # decode attention: PDL + cluster barrier (DSMEM merge)
}


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
@pytest.mark.parametrize("obj", sorted(EXPECT))
def test_hopper_mnemonics_present(built_lib, obj):
    sass = subprocess.run(["cuobjdump", "-sass", os.path.join(ROOT, "llmlb_b200", "_build", obj)], capture_output=True, text=True, timeout=600).stdout
    assert "sm_90a" in sass
    for pat, least in EXPECT[obj].items():
        n = len(re.findall(pat, sass))
        assert n >= least, "%s: %s occurs %d times, expected >= %d" % (obj, pat, n, least)
    if obj in ("gemm_tc.o", "gemm_tc2.o", "attention_tc.o"):
        assert not re.search(r"\bHMMA\b", sass), obj    # the wgmma kernels carry no mma.sync
