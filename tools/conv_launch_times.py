"""Per-launch device durations of the conv stack on the GPU: runs a few warm-up steps of a bench.py workload, then ONE step
under torch.profiler (CUDA activity only, a run of its own), and prints every conv kernel of that step in launch order in the
launch-list format tools/per_layer_roofline.py reads:

  python tools/conv_launch_times.py [workload] [out.txt]      # default config2, stdout

The header lines (starting with '#') name the card, its power limit and SM clock as read in the same run.  Durations are
from the CUDA activity trace of a step whose launches run back to back (L2 warm between producer and consumer layers), so
they add up to the step's conv time, unlike cold-cache replays."""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # the query is informational only
        q = f"nvidia-smi unavailable ({e})"
    return q


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile
    from bench import WORKLOADS
    from funcodec_b200 import get_config, init_state_dict
    from funcodec_b200.encodec import B200Encodec, _ptr

    workload = sys.argv[1] if len(sys.argv) > 1 else "config2"
    out = open(sys.argv[2], "w") if len(sys.argv) > 2 else sys.stdout
    assert torch.cuda.is_available(), "conv_launch_times.py needs a GPU"
    cfg_name, B, L, bw = WORKLOADS[workload]
    cfg = get_config(cfg_name)
    dev = torch.device("cuda", 0)
    model = B200Encodec(cfg, init_state_dict(cfg, 0), str(dev))
    n_q = cfg.num_quantizers_for_bandwidth(bw)
    Tf = cfg.frames(L)
    assert min(L, cfg.decoded_length(Tf)) == L, "round-trip workloads only"
    g = torch.Generator().manual_seed(1236)
    wav = (0.1 * torch.randn(B, L, generator=g)).to(dev)
    codes = torch.empty((n_q, B, Tf), dtype=torch.int64, device=dev)
    recon = torch.empty((B, 1, L), dtype=torch.float32, device=dev)

    def step():
        model._ck(model._lib.fcb_roundtrip(model._h, _ptr(wav), B, L, n_q, 1, _ptr(codes), None, None, None, _ptr(recon),
                                           model._stream()), "fcb_roundtrip")

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    kern = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    conv = [e for e in kern if "conv1d" in e["name"] or "conv2d" in e["name"]]
    print(f"# {workload}: {cfg_name}, B = {B}, {L} samples per clip; one step under torch.profiler (CUDA activity)", file=out)
    print(f"# card: {card_info()}   (name, power limit, SM clock, max SM clock)", file=out)
    print(f"# {len(kern)} kernels in the step, {len(conv)} conv launches, {sum(e['dur'] for e in conv) / 1e3:.3f} ms summed", file=out)
    for i, e in enumerate(conv):
        grid = "(" + ", ".join(str(x) for x in e.get("args", {}).get("grid", [])) + ")"
        print(f"  id {i:6d} {e['dur']:10.1f} us grid {grid:>18s} {e['name'].split('(')[0][-60:]}", file=out)


if __name__ == "__main__":
    main()
