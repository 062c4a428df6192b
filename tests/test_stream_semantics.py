"""The causality that chunked streaming rests on, pinned on the reference algorithm (the CPU oracle, itself pinned on the
unmodified reference): for a causal stack, the whole-clip run on a prefix of at least F_min frames gives the same codes and
waveform as the same span of the whole-clip run on the full clip, and F_min - 1 frames do not.  CPU only."""
import ctypes
import dataclasses
import os
import re

import numpy as np
import pytest
import torch

from funcodec_b200 import _capi, get_config, init_state_dict
from funcodec_b200.config import PRESETS
from oracle import encodec_oracle as O
from parity_utils import assert_codes_parity
from test_oracle_golden import test_model_inference as _pin_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_min_first_frames_of_every_causal_preset():
    """F_min = max over convs of ceil((p + 1) / input rows per frame): 7 for every causal preset, set by the k7 convs at frame
    rate (the final encoder conv and the first decoder conv)."""
    causal = [c for c in PRESETS.values() if c.causal]
    assert {"soundstream_16k_n32_ds320", "soundstream_causal_small", "causal_lstm_small"} <= {c.name for c in causal}
    for cfg in causal:
        assert cfg.stream_min_first_frames() == 7, cfg.name
        hist = cfg.stream_history()
        assert max(-(-(p + 1) // n) for p, n in hist) == 7
        assert (6, 1) in hist                                          # k7 at frame rate
        assert max(p for p, _ in hist) == max(6, (cfg.residual_kernel_size - 1) * cfg.dilation_base ** (cfg.n_residual_layers - 1),
                                              max(cfg.ratios))


@pytest.mark.parametrize("name", ["soundstream_causal_small", "causal_lstm_small"])
def test_prefix_of_min_first_frames_is_the_whole_clip(name):
    cfg = dataclasses.replace(get_config(name), audio_normalize=False)     # the stream's scale is given, not measured
    sd = init_state_dict(cfg, 5)
    o = O.OracleEncodec.from_config(sd, cfg)
    hop, fmin, F = cfg.hop_length, cfg.stream_min_first_frames(), 30
    g = torch.Generator().manual_seed(9)
    wav = 0.1 * torch.randn(2, F * hop, generator=g)
    whole = o.inference(wav, need_recon=True)
    for f in (fmin, fmin + 4):
        pre = o.inference(wav[:, :f * hop], need_recon=True, want_margin=True)
        res = assert_codes_parity(pre["code_indices"][0].numpy(), whole["code_indices"][0][:, :, :f].numpy(),
                                  pre["margins"].numpy(), 2e-3, what=f"{name} prefix {f}")
        ok = ~(res["first_stage"] >= 0).any(axis=1)
        assert ok.any()
        for b in np.nonzero(ok)[0]:
            d = (pre["recon_speech"][b] - whole["recon_speech"][b, :, :f * hop]).abs().max().item()
            assert d <= 1e-5, (name, f, b, d)
    # one frame less: some conv pads a row that the whole clip reads from the signal
    pre = o.inference(wav[:, :(fmin - 1) * hop], need_recon=True)
    d = (pre["recon_speech"] - whole["recon_speech"][:, :, :(fmin - 1) * hop]).abs().max().item()
    same_codes = torch.equal(pre["code_indices"][0], whole["code_indices"][0][:, :, :fmin - 1])
    assert d > 1e-4 or not same_codes, (name, d)


def test_oracle_matches_causal_lstm_golden(golden_dir):
    """The {weight_norm, causal, SLSTM} fixture generated from the unmodified reference (tools/gen_golden_norms.py)."""
    _pin_model(golden_dir, "model_causal_lstm_small.npz")


def test_stream_symbols_exported_and_declared():
    hdr = open(os.path.join(ROOT, "include", "funcodec_b200.h")).read()
    names = ["fcb_stream_min_first_frames", "fcb_stream_create", "fcb_stream_encode", "fcb_stream_decode_codes",
             "fcb_stream_decode_emb", "fcb_stream_reset", "fcb_stream_destroy"]
    lib = ctypes.CDLL(_capi.LIB_PATH)
    for n in names:
        assert re.search(r"FCB_API\s+[\w\s\*]+?\b" + n + r"\s*\(", hdr), n
        assert n in _capi.SYMBOLS and hasattr(lib, n), n
