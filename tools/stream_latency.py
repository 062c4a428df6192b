"""Latency of chunked streaming (encode_stream / decode_stream) on soundstream_16k_n32_ds320: per call, device time (CUDA
events), host wall time including a synchronise, kernel launches, and the real-time factor (audio seconds / wall seconds).
Chunks of 1 frame (20 ms) and 8 frames after a first chunk of F_min frames; encoder and decoder streams are timed separately.
Prints the card name and power limit with the numbers.  Needs a GPU.

    python tools/stream_latency.py [--batches 1 64 256] [--calls 50] [--warmup 10] [--json OUT]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from funcodec_b200 import get_config, init_state_dict  # noqa: E402
from funcodec_b200.encodec import B200Encodec  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def time_calls(model, push, chunk, calls, warmup):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(warmup):
        push(chunk)
    torch.cuda.synchronize()
    dev, wall = [], []
    n0 = model.launch_count()
    for _ in range(calls):
        t0 = time.perf_counter()
        ev0.record()
        push(chunk)
        ev1.record()
        torch.cuda.synchronize()
        wall.append(time.perf_counter() - t0)
        dev.append(ev0.elapsed_time(ev1) / 1e3)
    launches = (model.launch_count() - n0) / calls
    dev.sort()
    wall.sort()
    return dev[len(dev) // 2], wall[len(wall) // 2], launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 64, 256])
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stream_latency.py needs a GPU"
    cfg = get_config("soundstream_16k_n32_ds320")
    model = B200Encodec(cfg, init_state_dict(cfg, 0), "cuda:0")
    hop, fmin, D = cfg.hop_length, cfg.stream_min_first_frames(), cfg.dimension
    dev_name = card()
    print(f"# {dev_name}; {cfg.name}, hop {hop} samples = {hop / cfg.sample_rate * 1e3:.0f} ms", flush=True)
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for B in args.batches:
        scale = torch.ones(B, device="cuda")
        for f in args.frames:
            wav = 0.1 * torch.randn(B, f * hop, device="cuda", generator=g)
            first = 0.1 * torch.randn(B, fmin * hop, device="cuda", generator=g)
            tok = torch.randint(0, cfg.codebook_size, (B, f, cfg.num_quantizers), device="cuda", generator=g)
            es = model.encode_stream(B, scale)
            es.push(first)
            enc = time_calls(model, es.push, wav, args.calls, args.warmup)
            ds = model.decode_stream(B, scale)
            ds.push_emb(torch.zeros(B, fmin, D, device="cuda"))
            emb = 0.1 * torch.randn(B, f, D, device="cuda", generator=g)
            dec = time_calls(model, ds.push_emb, emb, args.calls, args.warmup)
            dsc = model.decode_stream(B, scale)
            dsc.push_codes(torch.zeros(B, fmin, cfg.num_quantizers, dtype=torch.int64, device="cuda"))
            decc = time_calls(model, dsc.push_codes, tok, args.calls, args.warmup)
            audio = f * hop / cfg.sample_rate
            for kind, (d, w, n) in (("encode", enc), ("decode_emb", dec), ("decode_codes", decc)):
                # real-time factor per stream (audio seconds of one clip / wall seconds) and over the batch
                r = dict(kind=kind, B=B, frames=f, device_ms=d * 1e3, wall_ms=w * 1e3, launches=n, rtf=audio / w,
                         rtf_batch=B * audio / w)
                rows.append(r)
                print(f"{kind:12s} B={B:4d} chunk={f} frames: device {r['device_ms']:.3f} ms, wall {r['wall_ms']:.3f} ms, "
                      f"{n:.0f} launches, real-time factor {r['rtf']:.1f} per clip, {r['rtf_batch']:.0f} over the batch",
                      flush=True)
            es.close(); ds.close(); dsc.close()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(dict(card=dev_name, preset=cfg.name, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
