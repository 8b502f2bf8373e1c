#!/usr/bin/env python
"""Static audit of libpn2_b200.so (no GPU needed): per kernel, registers / shared memory / spills from
`cuobjdump -res-usage` and the count of the SASS opcodes the design relies on (warp reductions, packed
FP32x2, vector atomics, async cluster stores, barriers).  Writes profiles/r2_sass_audit.txt."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pointnet2_b200", "libpn2_b200.so")
# (label, regex on the opcode) — first match wins
WATCH = [("CREDUX", r"^CREDUX"), ("REDUX", r"^REDUX"), ("FADD2", r"^FADD2"), ("FMUL2", r"^FMUL2"), ("FFMA2", r"^FFMA2"), ("FFMA", r"^FFMA"),
         ("FMNMX", r"^FMNMX"), ("FSETP", r"^FSETP"), ("REDG.F32x4", r"^REDG.*F32x4"), ("REDG.F32", r"^REDG"), ("ATOMG", r"^ATOMG"),
         ("ATOMS", r"^ATOMS"), ("STAS(st.async)", r"^STAS"), ("SYNCS(mbarrier)", r"^SYNCS"), ("UCGABAR(cluster barrier)", r"^UCGABAR"),
         ("PREEXIT(griddepcontrol.launch_dependents)", r"^PREEXIT"), ("ACQBULK(griddepcontrol.wait)", r"^ACQBULK"), ("BAR.SYNC", r"^BAR"), ("LDS.128", r"^LDS.*128"), ("LDS.64", r"^LDS.*64"), ("LDS", r"^LDS"), ("STS", r"^STS"),
         ("LDG.128", r"^LDG.*128"), ("STG.128", r"^STG.*128"), ("LDG", r"^LDG"), ("STG", r"^STG"), ("SHFL", r"^SHFL"), ("VOTE", r"^VOTE"),
         ("POPC", r"^POPC"), ("MUFU", r"^MUFU"), ("LDL", r"^LDL"), ("STL", r"^STL")]
SHOW = ["fps_cta_kernel<16, 256, 0, false>", "fps_cta_kernel<16, 256, 1, false>", "fps_cta_kernel<16, 256, 1, true>", "fps_cta_kernel<32, 256, 1, false>", "fps_cluster_kernel<16, 128, 16, 1, false>", "fps_cluster_kernel<32, 128, 32, 0, false>", "fps_cluster_kernel<32, 128, 32, 1, false>", "fps_cluster_kernel<32, 512, 16, 1, false>",
        "fps_cluster_big_kernel<52, 512, 16, 0, false>", "fps_cluster_big_kernel<52, 512, 16, 1, false>",
        "ball_group_kernel", "knn_kernel", "ball_query_kernel<16>", "bq_grid_build_kernel", "bq_grid_query_kernel",
        "group_rows_vec4_kernel<32, 4>", "group_narrow_kernel<false, float>", "group_rows_kernel<32, true, float>", "group_concat_vec_kernel<16, 2>",
        "group_point_grad_vec4_kernel<unsigned int, float>", "group_point_grad_vec4_kernel<unsigned int, __nv_bfloat16>", "three_nn_kernel", "fp_front_kernel<1, float>", "fp_front_kernel<8, float>", "fp_front_kernel<8, unsigned short>", "group_rows_kernel<32, true, unsigned short>",
        "three_interp_vec4_kernel<unsigned int, float, false, float4>", "three_interp_vec4_kernel<unsigned int, __nv_bfloat16, false, uint2>", "three_interp_grad_vec4_kernel<unsigned int>", "inv_build_kernel",
        "inv_gather_kernel<true, float>", "inv_long_kernel<true, float>", "inv_gather_kernel<true, unsigned short>", "inv_long_kernel<true, unsigned short>", "selection_sort_kernel", "prob_cumsum_kernel", "prob_search_kernel",
        "mbn_stats_kernel<float, 4, true>", "mbn_stats_kernel<__nv_bfloat16, 4, true>", "mbn_stats_kernel<float, 1, false>", "mbn_finalize_kernel",
        "mbn_norm_relu_kernel<float, 4, true>", "mbn_norm_relu_kernel<__nv_bfloat16, 4, true>", "mbn_bwd_sums_kernel<float, 4, true>",
        "mbn_bwd_sums_kernel<__nv_bfloat16, 4, true>", "mbn_bwd_finalize_kernel", "mbn_bwd_dx_kernel<float, 4, true>", "mbn_bwd_dx_kernel<__nv_bfloat16, 4, true>",
        "mbn_norm_relu_max_kernel<float, 4, true>", "mbn_norm_relu_max_kernel<__nv_bfloat16, 4, true>", "mbn_max_bwd_finalize_kernel<float>",
        "mbn_max_bwd_dx_kernel<float, 4, true>", "mbn_max_bwd_dx_kernel<__nv_bfloat16, 4, true>", "sa_mlp_keys_out_kernel<float>",
        "scene_count_kernel", "scene_scan_kernel", "scene_fill_kernel", "scene_merge_kernel<float>", "scene_merge_kernel<__nv_bfloat16>",
        "scene_merge_kernel<__half>", "crop_attempt_kernel", "crop_select_kernel", "shape_batch_kernel",
        "vscan_ray_kernel", "vscan_cell_kernel", "vscan_point_kernel", "vscan_select_kernel"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))


def main():
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    usage = {}
    cur = None
    for ln in res.splitlines():
        m = re.search(r"Function (\S+):", ln)
        if m:
            cur = m.group(1)
            continue
        if cur and "REG:" in ln:
            usage[cur] = {k: int(v) for k, v in re.findall(r"(REG|STACK|SHARED|LOCAL):(\d+)", ln)}
            cur = None
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    counts = collections.defaultdict(collections.Counter)
    total = collections.Counter()
    cur = None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d\s+)?([A-Za-z0-9_.]+)", ln)
        if cur and m:
            op = m.group(1)
            total[cur] += 1
            for label, rx in WATCH:
                if re.match(rx, op):
                    counts[cur][label] += 1
                    break
    names = demangle(sorted(usage))
    lines = ["# static audit of libpn2_b200.so (sm_90a): cuobjdump -res-usage + SASS opcode counts per kernel",
             "# REG = registers/thread, STACK = spill bytes, SHARED = static shared memory bytes; counts are static instruction counts",
             f"# {len(usage)} kernels in the library; spills (STACK > 0): "
             + (", ".join(f"{names[k]} ({v['STACK']} B)" for k, v in usage.items() if v.get("STACK", 0) > 0) or "none"), ""]
    for pat in SHOW:
        hits = [k for k in usage if pat in names[k].replace("pn2::", "").replace("(anonymous namespace)::", "")]
        for k in hits[:1]:
            u = usage[k]
            nice = re.sub(r"\(.*", "", names[k].replace("void ", "").replace("pn2::", "").replace("(anonymous namespace)::", ""))
            c = counts[k]
            lines.append(f"{nice}\n    REG {u.get('REG')}  STACK {u.get('STACK')}  SHARED {u.get('SHARED')}  instructions {total[k]}\n    "
                         + "  ".join(f"{w}:{c[w]}" for w, _ in WATCH if c[w]))
    out = os.path.join(ROOT, "profiles", "r2_sass_audit.txt")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as f:
        f.write("\n".join(lines) + "\n")
    print(open(out).read())


if __name__ == "__main__":
    sys.exit(main())
