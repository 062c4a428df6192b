"""Pins the FreqCodec (mag_phase, BASELINE config 4) oracle against vectors produced by the UNMODIFIED reference
(tools/gen_golden_freq.py).  CPU only.  The CUDA path for this variant is round-2 work; the oracle is ready for it."""
import os

import numpy as np
import torch

from oracle.freqcodec_oracle import OracleFreqCodec


def test_freqcodec_magphase_oracle_vs_reference(golden_dir):
    from funcodec_b200 import get_config, init_state_dict
    z = np.load(os.path.join(golden_dir, "freq_magphase_small.npz"))
    sd = init_state_dict(get_config(str(z["cfg_name"])), int(z["seed"]))
    assert abs(float(sum(v.double().abs().sum().item() for v in sd.values())) - float(z["sd_checksum"])) <= 1e-6 * float(z["sd_checksum"])
    o = OracleFreqCodec(sd, [tuple(r) for r in z["ratios"]])
    wav = torch.from_numpy(z["wav"])
    r = o.inference(wav, want_margin=True)
    assert r["features"].shape[1:3] == (3, 257)
    assert np.abs(r["encoder_out"].numpy() - z["encoder_out"]).max() <= 5e-6
    assert np.array_equal(r["code_indices"][0].numpy(), z["codes"].astype(np.int64))
    assert np.abs(r["code_embeddings"][0][0].numpy() - z["quant"]).max() <= 5e-6
    assert np.abs(r["code_embeddings"][0][1].numpy() - z["scale"]).max() <= 1e-7
    assert r["recon_speech"].shape == z["recon"].shape
    assert np.abs(r["recon_speech"].numpy() - z["recon"]).max() <= 5e-6


def test_freqcodec_config4_architecture_oracle_vs_reference(golden_dir):
    """BASELINE config 4's architecture (n_filters 32, D 128, K 1024, n_q 32, conv groups = 1) on a 0.5 s clip: the oracle
    against the unmodified reference FreqCodec (tools/gen_golden_freq.py); weights = init_state_dict(cfg, 0)."""
    from funcodec_b200 import get_config, init_state_dict
    z = np.load(os.path.join(golden_dir, "freq_magphase_config4_arch.npz"))
    cfg = get_config(str(z["cfg_name"]))
    sd = init_state_dict(cfg, int(z["seed"]))
    assert abs(float(sum(v.double().abs().sum().item() for v in sd.values())) - float(z["sd_checksum"])) <= 1e-6 * float(z["sd_checksum"])
    o = OracleFreqCodec(sd, list(zip(cfg.ratios_f, cfg.ratios)))
    r = o.inference(torch.from_numpy(z["wav"]), want_margin=True)
    assert np.abs(r["encoder_out"].numpy() - z["encoder_out"]).max() <= 1e-5
    assert np.array_equal(r["code_indices"][0].numpy(), z["codes"].astype(np.int64))
    assert np.abs(r["code_embeddings"][0][0].numpy() - z["quant"]).max() <= 1e-5
    assert r["recon_speech"].shape == z["recon"].shape
    assert np.abs(r["recon_speech"].numpy() - z["recon"]).max() <= 1e-5


def test_freq_layers_oracle_vs_reference_modules(golden_dir):
    """sconv2d / sconvtr2d / resblock2d against the reference MODULES SConv2d / SConvTranspose2d / SEANetResnetBlock2d
    (tools/gen_golden_freq_layers.py): every kernel / stride family, odd lengths, out_padding."""
    from oracle import freqcodec_oracle as FO
    z = np.load(os.path.join(golden_dir, "freq_layers.npz"))

    def sd_of(prefix):
        return {"L." + k[len(prefix) + 4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(prefix + ".sd.")}

    n = 0
    while f"conv{n}.x" in z.files:
        cin, cout, kf, kt, sf, st = [int(v) for v in z[f"conv{n}.meta"]]
        y = FO.sconv2d(torch.from_numpy(z[f"conv{n}.x"]), sd_of(f"conv{n}"), "L", stride=(sf, st))
        assert y.shape == z[f"conv{n}.y"].shape, (n, y.shape)
        assert np.abs(y.numpy() - z[f"conv{n}.y"]).max() <= 2e-6, n
        n += 1
    assert n == 6
    n = 0
    while f"convtr{n}.x" in z.files:
        cin, cout, sf, st, fl, fr, tl, tr = [int(v) for v in z[f"convtr{n}.meta"]]
        y = FO.sconvtr2d(torch.from_numpy(z[f"convtr{n}.x"]), sd_of(f"convtr{n}"), "L", (sf, st), ((fl, fr), (tl, tr)))
        assert y.shape == z[f"convtr{n}.y"].shape, (n, y.shape, z[f"convtr{n}.y"].shape)
        assert np.abs(y.numpy() - z[f"convtr{n}.y"]).max() <= 2e-6, n
        n += 1
    assert n == 3
    y = FO.resblock2d(torch.from_numpy(z["rb.x"]), sd_of("rb"), "L")
    assert np.abs(y.numpy() - z["rb.y"]).max() <= 2e-6


def _dense_convtr_weights(sd):
    """The engine's treatment of grouped transposed 2-D convs (engine.cu pack_convtr2d): block-diagonal dense weights
    [C_in][C_out]; plain convs are expanded by _dense_conv_weight once the consumer's C_in is known."""
    out = dict(sd)
    for k, w in sd.items():
        if w.dim() == 4 and k.endswith(".convtr.convtr.weight"):
            cin, cog = w.shape[:2]
            cout = sd[k.replace("weight", "bias")].shape[0]
            cig = cin // (cout // cog)
            dense = torch.zeros(cin, cout, *w.shape[2:])
            for ci in range(cin):
                dense[ci, (ci // cig) * cog:(ci // cig + 1) * cog] = w[ci]
            out[k] = dense
    return out


def _dense_conv_weight(w, cin):
    cout, cig = w.shape[:2]
    g = cin // cig
    cog = cout // g
    dense = torch.zeros(cout, cin, *w.shape[2:])
    for co in range(cout):
        dense[co, (co // cog) * cig:(co // cog + 1) * cig] = w[co]
    return dense


def test_freqcodec_grouped_convs_oracle_vs_reference(golden_dir):
    """conv_group_ratio / tr_conv_group_ratio > 0 (seanet_encoder.py:224,234,321; seanet_decoder.py:219,229,324): the oracle
    against the unmodified reference, and the dense block-diagonal expansion the engine uses against both."""
    from funcodec_b200 import get_config, init_state_dict
    z = np.load(os.path.join(golden_dir, "freq_magphase_small_grouped.npz"))
    cfg = get_config(str(z["cfg_name"]))
    assert cfg.conv_group_ratio > 0 and cfg.tr_conv_group_ratio > 0
    sd = init_state_dict(cfg, int(z["seed"]))
    assert sd["encoder.model.1.shortcut.conv.conv.weight"].shape[1] == cfg.n_filters // cfg.conv_groups(cfg.n_filters)
    ratios = list(zip(cfg.ratios_f, cfg.ratios))
    wav = torch.from_numpy(z["wav"])
    r = OracleFreqCodec(sd, ratios).inference(wav)
    assert np.abs(r["encoder_out"].numpy() - z["encoder_out"]).max() <= 5e-6
    assert np.array_equal(r["code_indices"][0].numpy(), z["codes"].astype(np.int64))
    assert np.abs(r["recon_speech"].numpy() - z["recon"]).max() <= 5e-6
    # dense expansion: every grouped weight becomes block-diagonal; the (group-inferring) oracle then runs groups = 1
    dense = _dense_convtr_weights(sd)
    from funcodec_b200.weights import state_dict_shapes
    dense_cfg = get_config("freq_small_grouped").__class__(**{**cfg.to_dict(), "conv_group_ratio": -1, "tr_conv_group_ratio": -1})
    for k, shp in state_dict_shapes(dense_cfg).items():
        if k.endswith(".conv.conv.weight") and len(shp) == 4:
            dense[k] = _dense_conv_weight(sd[k], shp[1])
            assert tuple(dense[k].shape) == tuple(shp)
        elif k.endswith(".convtr.convtr.weight"):
            assert tuple(dense[k].shape) == tuple(shp)
    r2 = OracleFreqCodec(dense, ratios).inference(wav)
    assert np.array_equal(r2["code_indices"][0].numpy(), z["codes"].astype(np.int64))
    assert np.abs(r2["recon_speech"].numpy() - z["recon"]).max() <= 1e-5


def test_freqcodec_ds640_ratios_oracle_vs_reference(golden_dir):
    """The ratio set of conf/freqcodec_mag_phase_16k_n32_600k_step_ds640.yaml ([[4, 2], [4, 1], [4, 2], [4, 1]]: a time stride
    in the first decoder stage / last encoder stage) against the unmodified reference; also the host-side frame arithmetic."""
    from funcodec_b200 import get_config, init_state_dict
    z = np.load(os.path.join(golden_dir, "freq_magphase_small_ds640.npz"))
    cfg = get_config(str(z["cfg_name"]))
    assert cfg.hop_length == 640
    sd = init_state_dict(cfg, int(z["seed"]))
    wav = torch.from_numpy(z["wav"])
    r = OracleFreqCodec(sd, list(zip(cfg.ratios_f, cfg.ratios))).inference(wav)
    assert r["encoder_out"].shape[1] == cfg.frames(wav.shape[-1]) == z["codes"].shape[-1]
    assert np.abs(r["encoder_out"].numpy() - z["encoder_out"]).max() <= 5e-6
    assert np.array_equal(r["code_indices"][0].numpy(), z["codes"].astype(np.int64))
    assert r["recon_speech"].shape == z["recon"].shape
    assert np.abs(r["recon_speech"].numpy() - z["recon"]).max() <= 5e-6
    assert min(wav.shape[-1], cfg.decoded_length(cfg.frames(wav.shape[-1]))) == z["recon"].shape[-1]


def test_freqcodec_config4_gr8_architecture_oracle_vs_reference(golden_dir):
    """BASELINE config 4 AS NAMED ("gr8": conv_group_ratio = tr_conv_group_ratio = 8 at the full widths): the oracle against
    the unmodified grouped reference FreqCodec (tools/gen_golden_freq_gr8.py); weights = init_state_dict(cfg, 0)."""
    from funcodec_b200 import get_config, init_state_dict
    z = np.load(os.path.join(golden_dir, "freq_magphase_config4_gr8_arch.npz"))
    cfg = get_config(str(z["cfg_name"]))
    assert cfg.conv_group_ratio == 8 and cfg.tr_conv_group_ratio == 8
    sd = init_state_dict(cfg, int(z["seed"]))
    assert abs(float(sum(v.double().abs().sum().item() for v in sd.values())) - float(z["sd_checksum"])) <= 1e-6 * float(z["sd_checksum"])
    # e.g. the 256-wide resblock: groups = 128 // 2 // 8 = 8 -> 16 input channels per group
    assert sd["encoder.model.10.block.1.conv.conv.weight"].shape[1] == 256 // cfg.conv_groups(128)
    o = OracleFreqCodec(sd, list(zip(cfg.ratios_f, cfg.ratios)))
    r = o.inference(torch.from_numpy(z["wav"]), want_margin=True)
    assert np.abs(r["encoder_out"].numpy() - z["encoder_out"]).max() <= 1e-5
    assert np.array_equal(r["code_indices"][0].numpy(), z["codes"].astype(np.int64))
    assert np.abs(r["code_embeddings"][0][0].numpy() - z["quant"]).max() <= 1e-5
    assert r["recon_speech"].shape == z["recon"].shape
    assert np.abs(r["recon_speech"].numpy() - z["recon"]).max() <= 1e-5
