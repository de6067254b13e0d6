"""Turn an `ncu --set full` capture of one diffusion step (23 launches; tools/ncu_capture.sh) into the committed artifacts:
profiles/<tag>_ncu_full_summary.csv (per launch) and, with --traffic, profiles/ncu_traffic.json (DRAM bytes per launch per kernel).
Input: the .ncu-rep or the raw-page CSV made from it.
    python tools/ncu_summary.py ncu_out/<tag>_cfg1_raw.csv <tag>_cfg1 --traffic"""
import csv, io, json, os, subprocess, sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METRICS = ["gpu__time_duration.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum",
           "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
           "lts__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
           "launch__registers_per_thread", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
           "l1tex__throughput.avg.pct_of_peak_sustained_elapsed"]
ORDER = ["embed_adaln"] + ["qkv_gemm", "attention", "outproj_gemm", "ff1_gemm", "ff2_gemm"] * 4 + ["head_gemm", "posterior_sample"]
UNIT = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}


def main():
    rep, tag = sys.argv[1], sys.argv[2]
    if rep.endswith(".csv"):
        out = open(rep).read()
    else:
        out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv", "--metrics", ",".join(METRICS)], capture_output=True, text=True).stdout
    out = out[out.index('"ID"'):]
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    assert len(data) == len(ORDER), f"expected {len(ORDER)} launches, got {len(data)}"
    cols = [hdr.index("Kernel Name")] + [hdr.index(m) for m in METRICS]

    def role_of(name):          # the capture window may start anywhere inside a step: name the launches by what they are
        if "embed_adaln" in name: return "embed_adaln"
        if "attention_kernel" in name: return "attention"
        if "posterior_sample" in name: return "posterior_sample"
        if "gemm_tc_kernel" in name:
            a = [x.strip().replace("(int)", "").replace("(bool)", "") for x in name[name.index("<") + 1:name.index(">")].split(",")]
            return {0: "qkv_gemm", 1: "ff1_gemm", 2: "head_gemm", 3: "ln_gemm"}[int(a[3])]   # <width, WG_M, stages, epilogue, mode>
        if "gemm_ln_kernel" in name: return "ln_gemm"
        return name[:24]
    roles = [role_of(r[cols[0]]) for r in data]
    # the out-projection and FF2 run the same LN GEMM kernel: the out-projection follows attention, FF2 follows FF1 (the window
    # is one whole step, so the first launch's predecessor is the last one)
    roles = [{"attention": "outproj_gemm", "ff1_gemm": "ff2_gemm"}[roles[i - 1]] if r == "ln_gemm" else r for i, r in enumerate(roles)]
    assert sorted(roles) == sorted(ORDER), f"launch window is not one whole step: {roles}"
    os.makedirs(os.path.join(REPO, "profiles"), exist_ok=True)
    with open(os.path.join(REPO, "profiles", f"{tag}_ncu_full_summary.csv"), "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["role"] + [hdr[c] for c in cols]); w.writerow([""] + [units[c] for c in cols])
        for role, r in zip(roles, data):
            w.writerow([role] + [r[c][:70] if c == cols[0] else r[c] for c in cols])
    ir, iw = hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
    acc = {}
    for role, r in zip(roles, data):
        b = float(r[ir]) * UNIT[units[ir]] + float(r[iw]) * UNIT[units[iw]]
        acc.setdefault(role, []).append(b)
    traffic = {k: round(sum(v) / len(v)) for k, v in acc.items()}
    print(json.dumps(traffic), "step total GB:", round(sum(sum(v) for v in acc.values()) / 1e9, 2))
    if "--traffic" not in sys.argv:
        return
    json.dump({"source": f"ncu --set full --clock-control none on tools/profile_step.py --steps 1 (B=1024): dram__bytes_read.sum + "
                         f"dram__bytes_write.sum, mean over the launches of one diffusion step (round {tag})",
               "dram_bytes_per_launch": traffic}, open(os.path.join(REPO, "profiles", "ncu_traffic.json"), "w"), indent=1)
    print(json.dumps(traffic))


if __name__ == "__main__":
    main()
