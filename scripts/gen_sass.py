#!/usr/bin/env python
"""Regenerate docs/sass/: one `cuobjdump -sass` listing per kernel of accl_b200/_C*.so (xz-compressed above 256 KB:
k_call and k_engine inline every collective body for every dtype and run to tens of MB of text) plus
docs/sass/HOT_LOOPS.md — the inner loops that matter, cut out of those listings around the instructions that prove
the Hopper / NVLink code paths (LDGMC = multimem.ld_reduce, multimem stores / reds, system-scope flag accesses,
HGMMA = wgmma.mma_async, UTMALDG / UTMAREDG = TMA load / reduce-add).

  python scripts/gen_sass.py            # needs the built extension; no GPU
"""
import glob
import lzma
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "docs", "sass")

# (title, kernel file stem, regex of the anchor instruction, lines before, lines after, comment)
EXCERPTS = [
    ("NVLS two-shot all-reduce: multimem.ld_reduce -> multimem.st (fp32, 8 x 16 B in flight per thread)", "k_call",
     r"LDGMC\.E\.ADD\.F32x4", 4, 40,
     "`LDGMC.E.ADD.F32x4.RN.STRONG.SYS` is `multimem.ld_reduce.relaxed.sys.global.add.v4.f32`: the NVSwitch returns the sum over "
     "all ranks' copies of the addressed 16 bytes; the stores that follow go to the multicast address (`multimem.st`), i.e. "
     "the reduced shard lands in every rank's result buffer.  No SM arithmetic on this path."),
    ("NVLS bf16 reduction with fp32 accumulation in the switch", "k_call", r"LDGMC\.E\.HPADD\.BF16x8", 2, 12,
     "`multimem.ld_reduce ... .add.acc::f32.v4.bf16x2`."),
    ("LL exchange: 8 payload bytes + 8 flag bytes per 16-byte store, consumer spins on the data", "k_call",
     r"ST\.E\.128\.STRONG\.SYS", 6, 24,
     "`st.volatile.global.v2.u64` to the peer's staging region (each 64-bit half = payload word | sequence number << 32) and the "
     "matching `LD.E.128.STRONG.SYS` poll loop on the local staging region: no fence, no separate flag."),
    ("system-scope release / acquire flags of the rendezvous meetings", "k_call", r"ST\.E\.STRONG\.SYS", 8, 16,
     "`st.release.sys` (MEMBAR.ALL.SYS + ST.E.STRONG.SYS) on the peer's sync pad and the `LD.E.STRONG.SYS` acquire spin."),
    ("persistent engine: command fetch / parked-call loop of the control CTA", "k_engine", r"NANOSLEEP", 20, 20,
     "the control CTA polls the command ring with `ld.acquire.sys`, steps every call in flight and backs off with NANOSLEEP "
     "only after 100 us without work."),
    ("wgmma GEMM: MMA issue loop", "k_plugin_gemm_rs_true_false_false_false", r"HGMMA\.64x256x16", 6, 30,
     "`wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16` from shared-memory descriptors, issued by each consumer "
     "warpgroup into its register accumulators."),
    ("wgmma GEMM, CTA pair: TMA loads", "k_plugin_gemm_rs_true_false_false_false", r"UTMALDG\.2D\.MULTICAST", 4, 10,
     "`cp.async.bulk.tensor.2d ... multicast::cluster`: each CTA of the pair loads half of the W tile into both CTAs."),
    ("wgmma GEMM epilogue: registers -> swizzled smem -> TMA reduce-add into the owner rank's shard", "k_plugin_gemm_rs_true_false_false_false",
     r"UTMAREDG\.2D\.ADD", 30, 6,
     "`UTMAREDG.2D.ADD` = `cp.reduce.async.bulk.tensor.2d ... .add`: the tile is added into "
     "peer memory over NVLink by the TMA unit (device API `reduce_scatter_emit_tile`)."),
    ("all-gather -> GEMM: MMA issue loop", "k_plugin_ag_gemm_false", r"HGMMA\.64x256x16", 6, 30,
     "the same m64n256k16 wgmma mainloop as the single-CTA GEMM -> reduce-scatter, on A tiles of own rows from the local "
     "shard and of peer rows from `gathered`."),
    ("all-gather -> GEMM: pull loop over the peer-mapped heap", "k_plugin_ag_gemm_false", r"LDG\.E\.128\.STRONG\.SYS", 4, 24,
     "`ld.volatile.global.v4.u32` from the peer's shard through its heap window, four loads in flight per thread before "
     "their `STG.E.NA.128` stores into the local `gathered` rows."),
    ("all-gather -> GEMM epilogue: registers -> swizzled smem -> TMA tensor store into C", "k_plugin_ag_gemm_false",
     r"UTMASTG\.2D", 30, 6,
     "`UTMASTG.2D` = `cp.async.bulk.tensor.2d.global.shared::cta.bulk_group`: the bf16 tile leaves shared memory for the "
     "local C through the TMA unit."),
    ("GEMM -> all-reduce: lazy per-tile signal to the owner", "k_plugin_gemm_rs_true_false_false_true", r"DEPBAR\.LE SB0, 0x0", 4, 40,
     "at the next tile's epilogue a consumer warp's lane 0 waits for its previous tile's reduce-adds to be performed "
     "(`cp.async.bulk.wait_group 0` = `DEPBAR.LE SB0, 0x0`), orders them before its generic accesses "
     "(`fence.proxy.async.global` = `FENCE.VIEW.ASYNC.G`) and adds 1 to the tile's counter in the owner's heap with "
     "`red.release.sys` (a system-scope `MEMBAR`, then `REDG.E.ADD.STRONG.SYS`)."),
    ("GEMM -> all-reduce: the owner's broadcast of a finished tile", "k_plugin_gemm_rs_true_false_false_true",
     r"LDG\.E\.128\.STRONG\.SYS", 4, 30,
     "warps 1-3 of the producer warpgroup, once a tile's counter holds all P ranks' arrivals: four `ld.volatile` 16-byte "
     "loads of the local tile in flight, then `STG.E.NA.128` stores of the same 16 bytes into every peer's C through the "
     "peer-mapped heap."),
    ("wgmma GEMM with a [K, N] weight: MMA issue loop", "k_plugin_gemm_rs_true_false_true_false", r"HGMMA\.64x256x16", 6, 30,
     "the same instruction with `.tnspB`: B is read MN-major from 64-column boxes of the [K, N] weight (an nn.Linear "
     "weight in its own backward pass), the descriptor advancing 2048 bytes per K=16 step."),
]


def main():
    so = glob.glob(os.path.join(ROOT, "accl_b200", "_C*.so"))
    if not so:
        sys.exit("build the extension first (python -m accl_b200.utils.build)")
    txt = subprocess.run(["cuobjdump", "-sass", so[0]], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"(?=\t\tFunction : )", txt)
    os.makedirs(OUT, exist_ok=True)
    for f in glob.glob(os.path.join(OUT, "*.sass*")):
        os.remove(f)
    listing = {}
    index = []
    for p in parts[1:]:
        name = p.split("\n")[0].split(": ")[1]
        dem = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()
        stem = re.sub(r"\(.*", "", dem).replace("accl::cuda::", "").replace("void ", "")
        stem = stem.replace("<", "_").replace(">", "").replace(", ", "_").replace("(bool)1", "true").replace("(bool)0", "false")
        listing[stem] = p
        ninstr = len(re.findall(r"/\*[0-9a-f]{4,}\*/\s+[A-Z@!]", p))
        if len(p) > (256 << 10):
            path = os.path.join(OUT, stem + ".sass.xz")
            with lzma.open(path, "wt", preset=6) as fh:
                fh.write(p)
        else:
            path = os.path.join(OUT, stem + ".sass")
            with open(path, "w") as fh:
                fh.write(p)
        ops = {}
        for m in re.finditer(r"\b(LDGMC[.\w]*|HGMMA[.\w]*|UTMALDG[.\w]*|UTMAREDG[.\w]*|"
                             r"REDG?\.E\.[.\w]*STRONG\.SYS|ST\.E\.128\.STRONG\.SYS|LD\.E\.128\.STRONG\.SYS|MEMBAR\.ALL\.SYS)", p):
            ops[m.group(1)] = ops.get(m.group(1), 0) + 1
        index.append((stem, dem, os.path.basename(path), ninstr, ops))
    with open(os.path.join(OUT, "README.md"), "w") as fh:
        fh.write("# SASS listings (cuobjdump -sass of accl_b200/_C*.so, sm_90a)\n\n"
                 "This index and `HOT_LOOPS.md` (the inner loops) are committed; the full per-kernel listings are not (k_call "
                 "and k_engine alone run to megabytes): `python scripts/gen_sass.py` writes them next to this file from a "
                 "build, no GPU needed; read the compressed ones with `xz -dc <file> | less`.\n\n"
                 "| kernel | listing | instructions | opcodes of interest |\n|---|---|---|---|\n")
        for stem, dem, path, n, ops in sorted(index):
            o = ", ".join(f"`{k}` x{v}" for k, v in sorted(ops.items()))
            fh.write(f"| `{dem[:110]}` | [{path}]({path}) | {n} | {o} |\n")
    with open(os.path.join(OUT, "HOT_LOOPS.md"), "w") as fh:
        fh.write("# Hot loops, cut out of the listings next to this file\n\n")
        for title, stem, rx, before, after, note in EXCERPTS:
            p = listing.get(stem)
            if p is None:
                continue
            lines = [ln for ln in p.split("\n") if re.search(r"/\*[0-9a-f]{4,}\*/\s+\S", ln)]
            idx = next((i for i, ln in enumerate(lines) if re.search(rx, ln)), None)
            fh.write(f"## {title}\n\n{note}\n\n")
            if idx is None:
                fh.write("(instruction not found in this build)\n\n")
                continue
            fh.write(f"`{stem}`:\n\n```\n")
            for ln in lines[max(0, idx - before): idx + after]:
                fh.write(re.sub(r"\s+/\* 0x[0-9a-f]+ \*/\s*$", "", ln).rstrip() + "\n")
            fh.write("```\n\n")
    print("wrote", len(index), "listings to", OUT)


if __name__ == "__main__":
    main()
