#!/usr/bin/env python
"""Summarise the SASS of the BUILT extension (`acco_b200/_C.so`, sm_90a) in `docs/sass/mnemonics.json`.

    python tools/dump_sass.py              # rewrite the summary
    python tools/dump_sass.py --listings   # also write the full listings to docs/sass/*.sass (large; not kept in git)
    python tools/dump_sass.py --check      # exit 1 if the committed summary does not describe the built binary

The summary counts, per listed kernel, the SASS mnemonics that show the Hopper-native path: `HGMMA` = wgmma.mma_async,
`UTMALDG` / `UTMASTG` = TMA load / store, `SYNCS` = mbarrier operations, `USETMAXREG` = setmaxnreg, `REDG` = per-element atomic
adds, `LDGMC` = multimem.ld_reduce, `QGMMA` = wgmma.mma_async on FP8 operands ...  `tests/test_sass_listings.py` runs the --check so a stale summary cannot be committed."""
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
    "gemm_pingpong_tn.sass": "_ZN9acco_gemm20gemm_pingpong_kernelILi0EEEvNS_6ParamsE",     # forward: ping-pong schedule
    "gemm_pingpong_nn.sass": "_ZN9acco_gemm20gemm_pingpong_kernelILi1EEEvNS_6ParamsE",     # dgrad: ping-pong schedule
    "rs_adam_ag_multimem_bf16.sass": "_ZN4acco17rs_adam_ag_kernelI13__nv_bfloat16S1_Li2ELb0ELb0EEEvNS_11RoundParamsE",
    "rs_adam_ag_p2p_bf16.sass": "_ZN4acco17rs_adam_ag_kernelI13__nv_bfloat16S1_Li1ELb0ELb0EEEvNS_11RoundParamsE",
    "rs_adam_ag_multimem_bf16_nodecay.sass": "_ZN4acco17rs_adam_ag_kernelI13__nv_bfloat16S1_Li2ELb0ELb1EEEvNS_11RoundParamsE",   # no_decay_1d
    "rs_adam_ag_local_bf16_nodecay.sass": "_ZN4acco17rs_adam_ag_kernelI13__nv_bfloat16S1_Li0ELb0ELb1EEEvNS_11RoundParamsE",
    "round_gate.sass": "_ZN4acco17round_gate_kernelENS_11RoundParamsE",
    "round_norm_multimem_bf16.sass": "_ZN4acco17round_norm_kernelI13__nv_bfloat16Li2EEEvNS_11RoundParamsEPff",   # max_grad_norm
    "round_norm_local_bf16.sass": "_ZN4acco17round_norm_kernelI13__nv_bfloat16Li0EEEvNS_11RoundParamsEPff",
    "attn_fwd_wgmma.sass": "_ZN9acco_attn15attn_fwd_kernelILb0EEEvNS_9FwdParamsE",
    "attn_fwd_wgmma_seg.sass": "_ZN9acco_attn15attn_fwd_kernelILb1EEEvNS_9FwdParamsE",      # document-masked (packed rows)
    "attn_bwd_mma.sass": "_ZN9acco_attn15attn_bwd_kernelILb0EEEvNS_9BwdParamsE",
    "attn_bwd_mma_seg.sass": "_ZN9acco_attn15attn_bwd_kernelILb1EEEvNS_9BwdParamsE",
    "gemm_fp8_bn128_e4m3.sass": "_ZN9acco_gemm15gemm_fp8_kernelILi128ELi1EEEvNS_6ParamsE",     # train.fp8: forward
    "gemm_fp8_bn128_e5m2.sass": "_ZN9acco_gemm15gemm_fp8_kernelILi128ELi2EEEvNS_6ParamsE",     # dgrad / wgrad
    "fp8_amax.sass": "_ZN8acco_fp815fp8_amax_kernelEPK5uint4xPj",
    "fp8_cast_e4m3.sass": "_ZN8acco_fp815fp8_cast_kernelILi0EEEvPK13__nv_bfloat16PKjiPhS6_Pfii",
    "embedding_bwd.sass": "_ZN4acco20embedding_bwd_kernelEP13__nv_bfloat16PKxS3_PKS0_ii",        # one write per row: no REDG
    # grad_accum_dtype=fp32: wgrad / FP8 wgrad / embedding backward adding into fp32 gradient accumulators
    "gemm_wgmma_bn128_tt_f32acc.sass": "_ZN9acco_gemm18gemm_f32acc_kernelILi128EEEvNS_6ParamsE",
    "gemm_wgmma_bn256_tt_f32acc.sass": "_ZN9acco_gemm18gemm_f32acc_kernelILi256EEEvNS_6ParamsE",
    "gemm_fp8_bn128_e5m2_f32acc.sass": "_ZN9acco_gemm22gemm_fp8_f32acc_kernelILi128ELi2EEEvNS_6ParamsE",
    "embedding_bwd_f32.sass": "_ZN4acco20embedding_bwd_kernelEPfPKxS2_PK13__nv_bfloat16ii",
    # cross-entropy <kSmooth, kZ>: label smoothing and z-loss (train.z_loss_weight) add no pass over the logits (MUFU.EX2 counts)
    "ce_fwd.sass": "_ZN4acco13ce_fwd_kernelILb0ELb0EEEvPK13__nv_bfloat16PKxPfS6_iixfff",
    "ce_fwd_smooth.sass": "_ZN4acco13ce_fwd_kernelILb1ELb0EEEvPK13__nv_bfloat16PKxPfS6_iixfff",
    "ce_fwd_z.sass": "_ZN4acco13ce_fwd_kernelILb0ELb1EEEvPK13__nv_bfloat16PKxPfS6_iixfff",
    "ce_fwd_smooth_z.sass": "_ZN4acco13ce_fwd_kernelILb1ELb1EEEvPK13__nv_bfloat16PKxPfS6_iixfff",
    "ce_reduce.sass": "_ZN4acco16ce_reduce_kernelILb0EEEvPKfPKxPfS5_xxS2_S5_f",
    "ce_reduce_z.sass": "_ZN4acco16ce_reduce_kernelILb1EEEvPKfPKxPfS5_xxS2_S5_f",
    "ce_bwd.sass": "_ZN4acco13ce_bwd_kernelILb0ELb0EEEvP13__nv_bfloat16PKxPKfS6_iixfff",
    "ce_bwd_smooth.sass": "_ZN4acco13ce_bwd_kernelILb1ELb0EEEvP13__nv_bfloat16PKxPKfS6_iixfff",
    "ce_bwd_z.sass": "_ZN4acco13ce_bwd_kernelILb0ELb1EEEvP13__nv_bfloat16PKxPKfS6_iixfff",
    "ce_bwd_smooth_z.sass": "_ZN4acco13ce_bwd_kernelILb1ELb1EEEvP13__nv_bfloat16PKxPKfS6_iixfff",
    # knowledge distillation <kT1> (train.distill_teacher): one pass over both rows forward, one more backward
    "kd_fwd.sass": "_ZN4acco13kd_fwd_kernelILb0EEEvPK13__nv_bfloat16S3_PKxPfS6_xiixf",
    "kd_fwd_t1.sass": "_ZN4acco13kd_fwd_kernelILb1EEEvPK13__nv_bfloat16S3_PKxPfS6_xiixf",
    "kd_reduce.sass": "_ZN4acco16kd_reduce_kernelEPKfPKxPfS4_S4_xxff",
    "kd_bwd.sass": "_ZN4acco13kd_bwd_kernelILb0EEEvP13__nv_bfloat16PKS1_PKxPKfS8_xiixfff",
    "kd_bwd_t1.sass": "_ZN4acco13kd_bwd_kernelILb1EEEvP13__nv_bfloat16PKS1_PKxPKfS8_xiixfff",
    # DPO (train.dpo_beta): one pass over the policy and reference rows forward, one over the policy backward
    "dpo_fwd.sass": "_ZN4acco14dpo_fwd_kernelEPK13__nv_bfloat16S2_PKxPfS5_iix",
    "dpo_reduce.sass": "_ZN4acco17dpo_reduce_kernelEPKfPKxPfS4_S4_S4_iixf",
    "dpo_bwd.sass": "_ZN4acco14dpo_bwd_kernelEP13__nv_bfloat16PKxPKfS5_S5_iiix",
    # SimPO / ORPO (train.simpo_beta / train.orpo_lambda): ce_fwd's pass, then this one-CTA reduction; the backward is dpo_bwd
    "simpo_reduce.sass": "_ZN4acco18pref_reduce_kernelILi0EEEvPKfPKxPfS5_S5_S5_iixff",
    "orpo_reduce.sass": "_ZN4acco18pref_reduce_kernelILi1EEEvPKfPKxPfS5_S5_S5_iixff",
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
    # FP8 wgmma (QGMMA) is listed only where it occurs, so the entries of the bf16 kernels keep their keys
    q = sum(1 for o in ops if o == "QGMMA" or o.startswith("QGMMA."))
    if q:
        c["QGMMA"] = q
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
