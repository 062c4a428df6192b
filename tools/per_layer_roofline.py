"""Per-launch roofline table of the conv stack: lines up the conv launches of one step in a launch list
(tools/conv_launch_times.py on the GPU, or tools/summarize_launches.py over an ncu capture) with the analytic per-launch work
(funcodec_b200.workload.conv_launches) and prints, per launch: shape, layer-boundary MB and GMAC for the batch, the duration,
achieved GB/s (and % of the measured HBM peak) and fp32-equivalent TFLOP/s.

  python tools/per_layer_roofline.py <launch_summary.txt> [preset] [B] [samples] [hbm_peak_GBps]

Durations from an ncu list are cold-cache and serialised (one kernel at a time, caches flushed between replays): they bound each launch
from above; the step-level number bench.py reports (all launches back to back, L2 warm between consumer and producer) is ~10 %
lower in sum.  Use the table for the SHAPE of the gap -- which launches sit far from the HBM line -- not for absolute claims."""
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from funcodec_b200 import get_config  # noqa: E402
from funcodec_b200.workload import conv_launches  # noqa: E402


def main():
    path = sys.argv[1]
    preset = sys.argv[2] if len(sys.argv) > 2 else "encodec_16k_n32_ds640"
    B = int(sys.argv[3]) if len(sys.argv) > 3 else 16
    L = int(sys.argv[4]) if len(sys.argv) > 4 else 160000
    peak = float(sys.argv[5]) if len(sys.argv) > 5 else 3350.0     # H100 SXM data sheet, HBM3
    durs = []
    for line in open(path):
        m = re.match(r"\s*id\s+\d+\s+([\d.]+) us grid\s+\(.*?\)\s+(.*)$", line)
        if m and "rvq" not in m.group(2):
            durs.append((float(m.group(1)), m.group(2).replace("void ", "").strip()))
    layers = conv_launches(get_config(preset), L)
    if len(durs) != len(layers):
        raise SystemExit(f"{len(durs)} conv launches in {path}, {len(layers)} in the model of {preset}")
    print(f"# {preset}, B = {B}, {L} samples per clip; durations from {os.path.basename(path)}; HBM peak {peak:.0f} GB/s")
    print(f"{'launch':22s} {'cin->cout k/s':>18s} {'T_out':>7s} {'MB':>8s} {'GMAC':>7s} {'us':>7s} {'GB/s':>7s} {'%HBM':>6s} {'TFLOP/s':>8s}  kernel")
    tot_b = tot_m = tot_t = 0.0
    groups = {}
    for (us, kern), l in zip(durs, layers):
        mb, gmac = l["bytes"] * B / 1e6, l["macs"] * B / 1e9
        gbs = mb / 1e3 / (us * 1e-6)
        tf = 2 * gmac / 1e3 / (us * 1e-6)
        print(f"{l['name']:22s} {l['cin']:>6d}->{l['cout']:<5d}{l['k']:>2d}/{l['s']:<2d} {l['T_out']:>7d} {mb:8.1f} {gmac:7.2f} {us:7.1f} "
              f"{gbs:7.0f} {100 * gbs / peak:6.1f} {tf:8.1f}  {kern}")
        tot_b += mb; tot_m += gmac; tot_t += us
        key = "T_out >= 10000 (C <= 128)" if l["T_out"] >= 10000 else ("T_out 2000 (C 256-512)" if l["T_out"] >= 1000 else "T_out 250 (C 1024 / LSTM inputs)")
        g = groups.setdefault(key, [0.0, 0.0, 0.0])
        g[0] += mb; g[1] += gmac; g[2] += us
    print(f"{'all 48 launches':22s} {'':>18s} {'':>7s} {tot_b:8.1f} {tot_m:7.2f} {tot_t:7.1f} {tot_b / 1e3 / (tot_t * 1e-6):7.0f} "
          f"{100 * tot_b / 1e3 / (tot_t * 1e-6) / peak:6.1f} {2 * tot_m / 1e3 / (tot_t * 1e-6):8.1f}")
    print("# by time resolution:")
    for key, (mb, gmac, us) in groups.items():
        print(f"#   {key:34s} {mb:8.1f} MB {gmac:7.2f} GMAC {us:8.1f} us ({100 * us / tot_t:4.1f} % of the conv time) "
              f"{mb / 1e3 / (us * 1e-6):6.0f} GB/s = {100 * mb / 1e3 / (us * 1e-6) / peak:4.1f} % HBM, {2 * gmac / 1e3 / (us * 1e-6):6.1f} TFLOP/s")


if __name__ == "__main__":
    main()
