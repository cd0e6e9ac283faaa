"""Turn the raw ncu CSV exports in a directory (default ncu_out/) into the summaries under profiles/.

    python tools/summarise_profiles.py [tag] [dir]"""
import collections
import csv
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G, P = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "ncu_out"), os.path.join(ROOT, "profiles")
tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
os.makedirs(P, exist_ok=True)

# ---- launch list: the last full step ------------------------------------------------
rows = [r for r in csv.reader(open(os.path.join(G, "launches.csv"))) if len(r) > 10]
hdr = rows[0]
ki, vi = hdr.index("Kernel Name"), hdr.index("Metric Value")
launches = [(r[ki], float(r[vi].replace(",", "")) / 1e3) for r in rows[1:]]
# steps start at the first forward layer kernel
step_starts = [i for i, (n, _) in enumerate(launches) if "pack_b_images_kernel" in n]     # one packing launch opens every step
a, b = (step_starts[-2], step_starts[-1]) if len(step_starts) >= 2 else (0, len(launches))
step = launches[a:b]
acc = collections.OrderedDict()
for n, t in step:
    short = n.split("(")[0].replace("void ", "").replace("ptrb200::", "")[:70]
    acc.setdefault(short, [0, 0.0])
    acc[short][0] += 1
    acc[short][1] += t
tot = sum(v[1] for v in acc.values())
with open(os.path.join(P, f"{tag}_launch_list.md"), "w") as f:
    f.write(f"# {tag}: every kernel launch of one LambdaRank training step (B=1024 x 256 x 136, default scorer)\n\n")
    f.write("`ncu --metrics gpu__time_duration.sum --clock-control none` (cold-cache, serialised: compare SHARES).\n")
    f.write(f"Launches in the step: {len(step)}; summed kernel time {tot:.1f} us.\n\n| kernel | launches | us | share |\n|---|---|---|---|\n")
    for n, (c, t) in sorted(acc.items(), key=lambda kv: -kv[1][1]):
        f.write(f"| `{n}` | {c} | {t:.1f} | {100 * t / tot:.1f}% |\n")
print(open(os.path.join(P, f"{tag}_launch_list.md")).read()[:2500])

# ---- full captures ---------------------------------------------------------------------
WANT = [("gpu__time_duration.sum", "duration us"), ("dram__bytes_read.sum", "dram read MB"), ("dram__bytes_write.sum", "dram write MB"),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM % of peak"), ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM % of peak"),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue active %"), ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe %"), ("smsp__inst_executed.sum", "warp instructions"),
        ("launch__registers_per_thread", "regs/thread"), ("launch__grid_size", "grid"), ("launch__block_size", "block"),
        ("launch__shared_mem_per_block_dynamic", "dyn smem KB")]
traffic = {}
NAME_MAP = {"rows_gemm_ws_kernel<0,": "rows_gemm_ws_fwd", "rows_gemm_ws_kernel<1,": "rows_gemm_ws_dgrad", "wgrad_tc_kernel": "wgrad_tc",
            "colstat4_kernel<1": "colstat_dy", "norm_bwd_apply4_kernel": "norm_bwd_apply4_kernel", "pairwise_bce_": "pairwise_bce_kernel<LAMBDA>",
            "approxndcg_kernel": "approxndcg_kernel", "lambdaloss_kernel": "lambdaloss_kernel", "listmle_kernel": "listmle_kernel"}
# file-name tag -> key of traffic.json for kernels that share one C++ name (the batched attention GEMM)
FILE_MAP = {"full_c_attn_qk": "attn_tc_qk", "full_c_attn_pv": "attn_tc_pv", "full_c_softmax": "softmax_rows_kernel",
            "full_c_softmax_bwd": "softmax_bwd_rows_kernel", "full_c_rows_gemm_tc": "rows_gemm_tc_fwd"}
WHAT = {"full_b": "config b (LambdaRank + pointwise MLP, B=1024 x 256 x 136)", "full_c": "config c (ApproxNDCG + list scorer L=3, B=64 x 512 x 136)",
        "full_d": "config d (LambdaLoss, B=256 x 1024 x 136)", "full_e": "config e (ListMLE bf16, B=1024 x 256 x 136)"}
with open(os.path.join(P, f"{tag}_kernels_full.md"), "w") as f:
    f.write(f"# {tag}: `ncu --set full --clock-control none --import-source on` of the heavy kernels\n\n")
    f.write("One launch each from the second training step of the named bench configuration (`tools/profile_r02.sh`).  dram bytes are per launch.\n\n")
    for fn in sorted(os.listdir(G)):
        if not (fn.startswith("full_") and fn.endswith("_raw.csv")):
            continue
        rws = list(csv.reader(open(os.path.join(G, fn))))
        if len(rws) < 3:
            continue
        h = rws[0]
        for r in rws[2:]:
            kn = r[h.index("Kernel Name")]
            what = next((v for k, v in WHAT.items() if fn.startswith(k)), "")
            f.write(f"## `{kn[:110]}`\n\n{fn[:-8]} -- {what}\n\n| metric | value |\n|---|---|\n")
            for m, label in WANT:
                if m in h:
                    f.write(f"| {label} | {r[h.index(m)]} |\n")
            stalls = sorted(((float(r[i].replace(",", "")), c) for i, c in enumerate(h) if "issue_stalled" in c and c.endswith("per_issue_active.ratio") and r[i]), reverse=True)[:5]
            if stalls:
                f.write("| top warp-stall reasons (warps stalled per issue-active cycle) | " +
                        ", ".join(f"{c.split('issue_stalled_')[1].split('_per_')[0]} {v:.2f}" for v, c in stalls) + " |\n")
            f.write("\n")
            if "dram__bytes_read.sum" in h:
                def mb(x):
                    return float(x.replace(",", ""))
                unit_r, unit_w = rws[1][h.index("dram__bytes_read.sum")], rws[1][h.index("dram__bytes_write.sum")]
                scale = {"Mbyte": 1e6, "Gbyte": 1e9, "Kbyte": 1e3, "byte": 1.0}
                tb = mb(r[h.index("dram__bytes_read.sum")]) * scale.get(unit_r, 1e6) + mb(r[h.index("dram__bytes_write.sum")]) * scale.get(unit_w, 1e6)
                fkey = next((v for k, v in FILE_MAP.items() if fn.startswith(k)), None)
                if fkey:
                    traffic.setdefault(fkey, tb)
                elif fn.startswith("full_b") or not fn.startswith("full_c"):
                    for key, nm in NAME_MAP.items():
                        if key in kn and nm not in traffic:
                            traffic[nm] = tb
json.dump(traffic, open(os.path.join(P, "traffic.json"), "w"), indent=1)
print(traffic)
