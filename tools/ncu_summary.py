#!/usr/bin/env python
"""Per-launch table from an `ncu --set full` report: duration, DRAM bytes read / written, DRAM GB/s and % of the DRAM peak,
tensor-pipe activity (% of peak sustained while active -- what BASELINE.json's north_star asks for on the matmuls),
SM throughput %, registers.  With --json it also writes {phase: DRAM bytes of the phase's launches in one step}.
Usage: python tools/ncu_summary.py prof.ncu-rep [--json traffic.json] > ncu_summary.txt
(`ncu -i <rep> --page raw --csv --print-units base` is the only thing it runs.)"""
import collections
import csv
import io
import json
import subprocess
import sys

# kernel name fragment -> bench.py phase
PHASE_OF = [("gather_ctx", "gather"), ("gather_sorted", "gather"), ("ctx_fused", "ctx_fwd"), ("EpiTanhStore", "ctx_fwd"),
            ("attn_fwd", "attn_fwd"), ("EpiExpSum", "logits"), ("EpiStoreLse", "logits"), ("expsum_", "xent"), ("true_logit", "xent"),
            ("scale_rows", "xent"), ("umma_gemm2_kernel<192, 6, 0, 1, umma::EpiStore>", "dv"),
            ("umma_gemm2_kernel<192, 6, 0, 0, umma::EpiStore>", "dx_gemm"), ("umma_gemm_kernel<192, 4, 1, 1, umma::EpiStore,", "dW"), ("xent_combine", "xent"), ("softmax_grad", "xent"),
            ("EpiAdam", "dY"), ("attn_bwd", "attn_bwd"), ("scatter_dx", "dx_scatter"), ("scatter_sorted", "dx_scatter"),
            ("scatter_inbox", "dx_scatter"), ("inbox_apply", "dx_scatter"), ("adam_rows", "adam_catchup"),
            ("mark_rows", "adam_catchup"), ("adam_sweep", "adam_sweep"), ("split_tf32", "split")]
TENSOR = ["sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
          "sm__pipe_tensor_op_hmma_cycles_active.avg.pct_of_peak_sustained_active",
          "sm__inst_executed_pipe_tensor.avg.pct_of_peak_sustained_active"]


def main(rep, json_out=None):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv", "--print-units", "base"], capture_output=True, text=True,
                         check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr = rows[0]
    ix = {h: i for i, h in enumerate(hdr)}
    col = lambda r, name: r[ix[name]]
    tcol = next((t for t in TENSOR if t in ix), None)

    def num(r, name, default=0.0):
        try:
            return float(col(r, name))
        except (KeyError, ValueError):
            return default
    print("%-72s %12s %4s %9s %10s %10s %9s %7s %8s %6s" % ("kernel", "grid", "regs", "us", "dram_rd_MB", "dram_wr_MB", "DRAM GB/s",
                                                             "dram%", "tensor%", "sm%"))
    per_phase = collections.defaultdict(float)
    data = rows[2:]
    # one step's worth of launches: from the first captured kernel up to (not including) its next occurrence
    key = lambda r: (col(r, "Kernel Name"), col(r, "Grid Size"))
    period = next((j for j in range(1, len(data)) if key(data[j]) == key(data[0])), len(data))
    for i, r in enumerate(data):
        full = col(r, "Kernel Name")
        name = full.replace("c2v::umma::", "").replace("c2v::", "").split("(CUtensorMap")[0].split("(float")[0][:72]
        us = num(r, "gpu__time_duration.sum") / 1e3
        rd, wr = num(r, "dram__bytes_read.sum"), num(r, "dram__bytes_write.sum")
        print("%-72s %12s %4s %9.1f %10.1f %10.1f %9.0f %7.1f %8.1f %6.1f" % (
            name, col(r, "Grid Size").replace(" ", ""), col(r, "launch__registers_per_thread"), us, rd / 1e6, wr / 1e6,
            (rd + wr) / max(us, 1e-9) / 1e3, num(r, "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
            num(r, tcol) if tcol else float("nan"), num(r, "sm__throughput.avg.pct_of_peak_sustained_elapsed")))
        if i < period:
            for frag, phase in PHASE_OF:
                if frag in full:
                    per_phase[phase] += rd + wr
                    break
    print("# tensor%% = %s" % (tcol or "not in this report"))
    if json_out:
        json.dump({k: round(v) for k, v in per_phase.items()}, open(json_out, "w"), indent=1)


if __name__ == "__main__":
    args = sys.argv[1:]
    jo = None
    if "--json" in args:
        i = args.index("--json")
        jo = args[i + 1]
        del args[i:i + 2]
    main(args[0], jo)
