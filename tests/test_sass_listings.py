"""The committed SASS evidence must describe the binary that is actually built (round-1 finding: a listing had gone stale after a
kernel change).  CPU-only: needs the built `acco_b200/_C.so` (``__graft_entry__.build()``) and `cuobjdump`."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_docs_sass_matches_built_extension():
    if not os.path.exists(os.path.join(ROOT, "acco_b200", "_C.so")) or shutil.which("cuobjdump") is None:
        pytest.skip("extension not built / cuobjdump missing")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "dump_sass.py"), "--check"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=300)
    assert p.returncode == 0, p.stdout[-3000:]


def test_hopper_native_mnemonics_present():
    """wgmma / TMA / setmaxnreg / multimem instructions are in the shipped kernels (docs/sass/mnemonics.json, tools/dump_sass.py)."""
    import json
    m = json.load(open(os.path.join(ROOT, "docs", "sass", "mnemonics.json")))
    for name in ("gemm_wgmma_bn256_tn.sass", "gemm_wgmma_bn256_nn.sass", "gemm_wgmma_bn128_tt.sass"):
        g = m[name]
        assert g["HGMMA"] > 0 and g["UTMALDG"] > 0 and g["UTMALDG.2D.MULTICAST"] > 0 and g["UTMASTG"] > 0 and g["USETMAXREG"] > 0, name
        assert g["HMMA"] == 0, name                          # no legacy mma.sync path
    assert m["rs_adam_ag_multimem_bf16.sass"]["LDGMC"] > 0   # multimem.ld_reduce
    a = m["attn_fwd_wgmma.sass"]                             # own attention forward: wgmma fed by a TMA ring
    assert a["HGMMA"] > 0 and a["UTMALDG"] > 0 and a["SYNCS"] > 0
