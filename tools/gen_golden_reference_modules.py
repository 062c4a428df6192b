"""Snapshot of the UNMODIFIED reference's model objects for the host-side integration tests (build container only):
tests/golden/reference_modules.json.

For every preset the tests map, the reference `Encodec` built by tools/ref_harness.py is recorded as a module tree (class
name, the option attributes integration.config_from_reference_model inspects, children in registration order) plus its
state_dict key -> shape map.  Also recorded: the state_dict key -> shape map of the reference's `use_ddp: false` quantizer
(core_vq.ResidualVectorQuantization).  tests/test_capi_symbols.py rebuilds stand-in objects from this file."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from ref_harness import build_reference_encodec, import_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "reference_modules.json")
PRESETS = ("encodec_16k_n32_ds320", "tiny_ds40", "soundstream_noncausal_small", "soundstream_causal_small", "weightnorm_lstm_small")
# attributes read by integration.config_from_reference_model / _check_module_options
ATTRS = ("causal", "trim_right_ratio", "pad_mode", "dilation", "skip", "alpha", "num_groups", "num_channels", "ratios",
         "q0_ds_ratio", "sampling_rate", "encoder_hop_length", "codebook_size", "audio_normalize", "segment_dur",
         "overlap_ratio", "codec_domain", "domain_conf", "input_proj", "input_act")


def _value(v):
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    if isinstance(v, (list, tuple)):
        vals = [_value(x) for x in v]
        return vals if all(x is not _SKIP for x in vals) else _SKIP
    if isinstance(v, dict):
        return {str(k): _value(x) for k, x in v.items()}
    return _SKIP


_SKIP = object()


def snap(mod):
    import torch.nn as nn
    attrs = {}
    for a in ATTRS:
        if a in mod._modules:
            continue                                     # a child module, recorded below
        if hasattr(mod, a):
            v = _value(getattr(mod, a))
            if v is not _SKIP:
                attrs[a] = v
    return {"type": type(mod).__name__, "attrs": attrs,
            "children": [[n, snap(c)] for n, c in mod.named_children() if isinstance(c, nn.Module)]}


def main():
    from funcodec_b200 import get_config
    out = {"models": {}}
    for name in PRESETS:
        m = build_reference_encodec(get_config(name))
        out["models"][name] = {"tree": snap(m), "state_dict": {k: list(v.shape) for k, v in m.state_dict().items()}}
    import_reference()
    from funcodec.modules.quantization.core_vq import ResidualVectorQuantization
    rvq = ResidualVectorQuantization(num_quantizers=3, dim=16, codebook_size=32, decay=0.99, kmeans_init=True, kmeans_iters=10,
                                     threshold_ema_dead_code=2, quantize_dropout=True, rand_num_quant=[1, 2, 3])
    out["use_ddp_false_rvq"] = {"num_quantizers": 3, "dim": 16, "codebook_size": 32,
                                "state_dict": {k: list(v.shape) for k, v in rvq.state_dict().items()}}
    with open(OUT, "w") as f:
        json.dump(out, f, separators=(",", ":"), sort_keys=False)
        f.write("\n")
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
