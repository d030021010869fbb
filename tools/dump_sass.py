#!/usr/bin/env python
"""Summarise the SASS of the BUILT extension (`acco_b200/_C.so`, sm_90a) in `docs/sass/mnemonics.json`.

    python tools/dump_sass.py              # rewrite the summary
    python tools/dump_sass.py --listings   # also write the full listings to docs/sass/*.sass (large; not kept in git)
    python tools/dump_sass.py --check      # exit 1 if the committed summary does not describe the built binary

The summary counts, per listed kernel, the SASS mnemonics that show the Hopper-native path: `HGMMA` = wgmma.mma_async,
`UTMALDG` / `UTMASTG` = TMA load / store, `SYNCS` = mbarrier operations, `USETMAXREG` = setmaxnreg, `REDG` = the split-K atomic
adds, `LDGMC` = multimem.ld_reduce ...  `tests/test_sass_listings.py` runs the --check so a stale summary cannot be committed."""
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "acco_b200", "_C.so")
OUT = os.path.join(ROOT, "docs", "sass")

KERNELS = {
    "gemm_wgmma_bn256_tn.sass": "_ZN9acco_gemm11gemm_kernelILi256ELi0ELi0EEEvNS_6ParamsE",
    "gemm_wgmma_bn256_nn.sass": "_ZN9acco_gemm11gemm_kernelILi256ELi0ELi1EEEvNS_6ParamsE",
    "gemm_wgmma_bn128_tt.sass": "_ZN9acco_gemm11gemm_kernelILi128ELi1ELi1EEEvNS_6ParamsE",
    "rs_adam_ag_multimem_bf16.sass": "_ZN4acco17rs_adam_ag_kernelI13__nv_bfloat16S1_Li2ELb0EEEvNS_11RoundParamsE",
    "rs_adam_ag_p2p_bf16.sass": "_ZN4acco17rs_adam_ag_kernelI13__nv_bfloat16S1_Li1ELb0EEEvNS_11RoundParamsE",
    "round_gate.sass": "_ZN4acco17round_gate_kernelENS_11RoundParamsE",
    "attn_fwd_wgmma.sass": "_ZN9acco_attn15attn_fwd_kernelENS_9FwdParamsE",
}
MNEMONICS = ["HGMMA", "UTMALDG", "UTMALDG.2D.MULTICAST", "UTMASTG", "UTMACMDFLUSH", "SYNCS", "USETMAXREG", "REDG", "LDGMC", "HMMA", "MUFU.SQRT",
             "MUFU.EX2", "CCTL"]


def listing(func: str) -> str:
    p = subprocess.run(["cuobjdump", "-sass", "-fun", func, SO], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0 or "Function :" not in p.stdout:
        raise RuntimeError(f"cuobjdump failed for {func}: {p.stdout[-300:]}")
    txt = p.stdout[p.stdout.index("Function :"):]
    return re.sub(r"/\* 0x[0-9a-f]{16} \*/", "", txt)       # drop the raw encodings: smaller, and stable across relinks


def count(txt: str) -> dict:
    ops = re.findall(r"^\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", txt, flags=re.M)
    c = {"instructions": len(ops)}
    for m in MNEMONICS:
        c[m] = sum(1 for o in ops if o == m or o.startswith(m + "."))
    # multimem.st shows up as a STG on the multicast address: count the .STRONG.SYS 128-bit stores as a proxy
    c["STG.E.128.STRONG.SYS"] = sum(1 for o in ops if o.startswith("STG.E") and "128" in o and "SYS" in o)
    return c


def main():
    check = "--check" in sys.argv
    if not os.path.exists(SO):
        print("acco_b200/_C.so is not built")
        return 2
    summary = {}
    for fname, func in KERNELS.items():
        txt = listing(func)
        summary[fname] = {"function": func, **count(txt)}
        if not check and "--listings" in sys.argv:
            with open(os.path.join(OUT, fname), "w") as f:
                f.write(txt)
    path = os.path.join(OUT, "mnemonics.json")
    if check:
        want = json.load(open(path))
        strip = lambda d: {k: v for k, v in (d or {}).items() if k != "instructions"}    # total count: informational (scheduling noise)
        bad = {k: (want.get(k), v) for k, v in summary.items() if strip(want.get(k)) != strip(v)}
        if bad:
            print("docs/sass is stale (run tools/dump_sass.py):", json.dumps(bad, indent=1)[:2000])
            return 1
        print("docs/sass matches the built extension")
        return 0
    json.dump(summary, open(path, "w"), indent=1)
    print(json.dumps(summary, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
