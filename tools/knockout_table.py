"""Lines up several per-launch lists of the same workload (tools/conv_launch_times.py, one per FCB_TC_DBG knock-out setting) and
prints, per conv launch: the duration under every setting, its change against the first list, and for the tensor-core launches
the time per (64-channel chunk, tap) weight slab of one CTA.  The last block sums the launches that stream their weights.

  python tools/knockout_table.py <preset> <B> <samples> <label>=<launch list> [<label>=<launch list> ...]

Per-slab time = duration x CTAs / tiles / slabs per tile, with tiles = B * ceil(T_out / 128) * (C_out / N), one CTA per SM (at most
132) and ceil(C_in / 64) * K slabs per tile.  A layer streams its weights unless it has a single n-tile (C_out == N) and at most
64 slabs (tc_plan in conv_tc.cu keeps such an image resident in shared memory)."""
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from funcodec_b200 import get_config  # noqa: E402
from funcodec_b200.workload import conv_launches  # noqa: E402

SMS = 132


def read_list(path):
    durs, header = [], []
    for line in open(path):
        if line.startswith("# card:"):
            header.append(line[2:].strip())
        m = re.match(r"\s*id\s+\d+\s+([\d.]+) us grid\s+\(.*?\)\s+(.*)$", line)
        if m:
            durs.append((float(m.group(1)), m.group(2).replace("void ", "").strip()))
    return durs, header


def main():
    preset, B, L = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    runs = [a.split("=", 1) for a in sys.argv[4:]]
    layers = conv_launches(get_config(preset), L)
    lists = []
    for label, path in runs:
        durs, header = read_list(path)
        if len(durs) != len(layers):
            raise SystemExit(f"{len(durs)} conv launches in {path}, {len(layers)} in the model of {preset}")
        lists.append(durs)
        print(f"# {label:>8s}: {os.path.basename(path)}; {' '.join(header)}")
    labels = [r[0] for r in runs]
    print(f"{'launch':22s} {'cin->cout k/s':>18s} {'T_out':>6s} {'N':>4s} {'tiles':>6s} {'slabs':>5s} {'w':>3s} "
          + " ".join(f"{l + ' us':>10s}" for l in labels) + " " + " ".join(f"{'d ' + l:>8s}" for l in labels[1:])
          + " " + " ".join(f"{l + ' us/slab':>13s}" for l in labels))
    streamed = [0.0] * len(runs)
    n_streamed = 0
    for i, l in enumerate(layers):
        kern = lists[0][i][1]
        m = re.search(r"conv1d_tc_kernel<(\d+)", kern)
        us = [d[i][0] for d in lists]
        delta = " ".join(f"{100 * (u - us[0]) / us[0]:+7.1f}%" for u in us[1:])
        if m:
            n = int(m.group(1))
            # a transposed conv (k = 2s) runs as a 2-tap conv over the input rows with s * C_out columns (engine.cu pack_convtr)
            up = ".up" in l["name"]
            t_rows, cols, taps = (l["T_out"] // l["s"], l["s"] * l["cout"], 2) if up else (l["T_out"], l["cout"], l["k"])
            tiles = B * ((t_rows + 127) // 128) * (cols // n)
            slabs = ((l["cin"] + 63) // 64) * taps
            resident = cols == n and slabs <= 64
            per_slab = " ".join(f"{u * min(SMS, tiles) / tiles / slabs:13.2f}" for u in us)
            tag = "res" if resident else "str"
            if not resident:
                n_streamed += 1
                streamed = [s + u for s, u in zip(streamed, us)]
            shape = f"{n:4d} {tiles:6d} {slabs:5d} {tag:>3s}"
        else:
            per_slab = ""
            shape = f"{'-':>4s} {'-':>6s} {'-':>5s} {'-':>3s}"
        print(f"{l['name']:22s} {l['cin']:>6d}->{l['cout']:<5d}{l['k']:>2d}/{l['s']:<2d} {l['T_out']:>6d} {shape} "
              + " ".join(f"{u:10.1f}" for u in us) + " " + delta + " " + per_slab)
    totals = [sum(d[i][0] for i in range(len(layers))) for d in lists]
    print(f"# all {len(layers)} launches:        " + "  ".join(f"{l} {t / 1e3:.3f} ms" for l, t in zip(labels, totals)))
    print(f"# {n_streamed} streamed-weight launches: " + "  ".join(
        f"{l} {s / 1e3:.3f} ms ({100 * (s - streamed[0]) / streamed[0]:+.1f} %)" for l, s in zip(labels, streamed)))


if __name__ == "__main__":
    main()
