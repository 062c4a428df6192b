"""GPU parity for the FreqCodec mag_phase variant (BASELINE config 4, SURVEY.md §8 rows R19-R20) through the C ABI:
golden vectors from the unmodified reference + the CPU oracle (oracle/freqcodec_oracle.py) on seeded inputs."""
import os
import zlib

import numpy as np
import pytest
import torch

from funcodec_b200 import get_config, init_state_dict
from oracle.freqcodec_oracle import OracleFreqCodec
from parity_utils import assert_codes_parity

pytestmark = pytest.mark.gpu

WAV_TOL = 1e-4
EMB_TOL = 5e-5
MARGIN = 2e-3
_M = {}


def _small(golden_dir):
    from funcodec_b200.encodec import B200Encodec
    if "small" not in _M:
        z = np.load(os.path.join(golden_dir, "freq_magphase_small.npz"))
        cfg = get_config(str(z["cfg_name"]))
        sd = init_state_dict(cfg, int(z["seed"]))
        assert abs(float(sum(v.double().abs().sum().item() for v in sd.values())) - float(z["sd_checksum"])) <= 1e-6 * float(z["sd_checksum"])
        _M["small"] = (z, cfg, sd, B200Encodec(cfg, sd, "cuda:0"), OracleFreqCodec(sd, list(zip(cfg.ratios_f, cfg.ratios))))
    return _M["small"]


def test_freq_golden(golden_dir):
    z, cfg, sd, model, oracle = _small(golden_dir)
    wav = torch.from_numpy(z["wav"])
    ora = oracle.inference(wav, want_margin=True)
    r = model.inference(wav, need_recon=True, need_encoder_out=True)
    enc = r["encoder_out"].cpu().numpy()
    assert enc.shape == z["encoder_out"].shape
    assert np.abs(enc - z["encoder_out"]).max() <= EMB_TOL, np.abs(enc - z["encoder_out"]).max()
    codes = r["code_indices"][0].cpu().numpy()
    res = assert_codes_parity(codes, z["codes"], ora["margins"].numpy(), MARGIN, min_exact_rate=0.9, what="freq golden")
    ok_clip = ~(res["first_stage"] >= 0).any(axis=1)
    recon = r["recon_speech"].cpu().numpy()
    assert recon.shape == z["recon"].shape
    for b in np.nonzero(ok_clip)[0]:
        assert np.abs(recon[b] - z["recon"][b]).max() <= WAV_TOL, np.abs(recon[b] - z["recon"][b]).max()
    # decode-only parity from the reference's quantized embeddings
    d = model.inference_decoding_emb(torch.from_numpy(z["quant"]))
    dref = oracle.decode_frame(torch.from_numpy(z["quant"]), None)
    assert tuple(d["recon_speech"].shape) == tuple(dref.shape)
    assert (d["recon_speech"].cpu() - dref).abs().max().item() <= WAV_TOL * 10      # un-scaled output (~10x amplitude)


@pytest.mark.parametrize("B,L", [(3, 160 * 21 + 5), (1, 160 * 40), (2, 160 * 37 + 159)])
def test_freq_seeded(golden_dir, B, L):
    """Ragged lengths incl. the case where the iSTFT yields fewer than L samples (even STFT frame count)."""
    z, cfg, sd, model, oracle = _small(golden_dir)
    g = torch.Generator().manual_seed(B * 1000 + L)
    wav = 0.1 * torch.randn(B, L, generator=g)
    ora = oracle.inference(wav, want_margin=True)
    r = model.inference(wav, need_recon=True, need_encoder_out=True)
    assert tuple(r["recon_speech"].shape) == tuple(ora["recon_speech"].shape)
    assert (r["encoder_out"].cpu() - ora["encoder_out"]).abs().max().item() <= EMB_TOL
    res = assert_codes_parity(r["code_indices"][0].cpu().numpy(), ora["code_indices"][0].numpy(), ora["margins"].numpy(),
                              MARGIN, min_exact_rate=0.9, what="freq seeded")
    ok_clip = ~(res["first_stage"] >= 0).any(axis=1)
    for b in np.nonzero(ok_clip)[0]:
        assert (r["recon_speech"][b].cpu() - ora["recon_speech"][b]).abs().max().item() <= WAV_TOL


def _full():
    from funcodec_b200.encodec import B200Encodec
    if "full" not in _M:
        cfg = get_config("freqcodec_magphase_16k_n32_ds320")
        sd = init_state_dict(cfg, 0)
        _M["full"] = (cfg, sd, B200Encodec(cfg, sd, "cuda:0"), OracleFreqCodec(sd, list(zip(cfg.ratios_f, cfg.ratios))))
    return _M["full"]


@pytest.mark.parametrize("tc2d", [7, 0, 1, 3])
def test_freq_full_config_shapes_and_oracle_spot_check(tc2d):
    """BASELINE config 4 architecture (repo YAML, groups = 1) on a short clip against the oracle, with every 2-D conv on
    the tensor-core path (use_tc2d = 7, the default), all on the SIMT kernel (0), and the intermediate class masks."""
    cfg, sd, model, oracle = _full()
    model.set_option("use_tc2d", tc2d)
    try:
        g = torch.Generator().manual_seed(4)
        wav = 0.1 * torch.randn(2, 8000, generator=g)
        if "full_ora" not in _M:
            _M["full_ora"] = oracle.inference(wav, want_margin=True)
        ora = _M["full_ora"]
        r = model.inference(wav, need_recon=True, need_encoder_out=True, need_sub_quants=False)
        assert tuple(r["code_indices"][0].shape) == (32, 2, 26)
        err = (r["encoder_out"].cpu() - ora["encoder_out"]).abs().max().item()
        print(f"use_tc2d={tc2d}: encoder_out max-abs err {err:.3e}")
        assert err <= EMB_TOL
        res = assert_codes_parity(r["code_indices"][0].cpu().numpy(), ora["code_indices"][0].numpy(), ora["margins"].numpy(),
                                  MARGIN, min_exact_rate=0.9, what="freq full")
        ok_clip = ~(res["first_stage"] >= 0).any(axis=1)
        for b in np.nonzero(ok_clip)[0]:
            assert (r["recon_speech"][b].cpu() - ora["recon_speech"][b]).abs().max().item() <= WAV_TOL
        # decode-only parity (no code flips involved): the oracle's quantized embeddings through the 2-D decoder
        quant = ora["code_embeddings"][0][0]
        d = model.inference_decoding_emb(quant)
        dref = oracle.decode_frame(quant, None)
        derr = (d["recon_speech"].cpu() - dref).abs().max().item()
        print(f"use_tc2d={tc2d}: decode-only max-abs err {derr:.3e}")
        assert derr <= WAV_TOL * 10                      # un-scaled output (~10x amplitude)
    finally:
        model.set_option("use_tc2d", 7)


def test_freq_config4_arch_golden(golden_dir):
    """The config-4 architecture against vectors of the UNMODIFIED reference FreqCodec (tools/gen_golden_freq.py,
    weights = init_state_dict(cfg, 0) loaded into the reference module)."""
    cfg, sd, model, oracle = _full()
    z = np.load(os.path.join(golden_dir, "freq_magphase_config4_arch.npz"))
    wav = torch.from_numpy(z["wav"])
    ora = oracle.inference(wav, want_margin=True)
    r = model.inference(wav, need_recon=True, need_encoder_out=True, need_sub_quants=False)
    assert np.abs(r["encoder_out"].cpu().numpy() - z["encoder_out"]).max() <= EMB_TOL
    res = assert_codes_parity(r["code_indices"][0].cpu().numpy(), z["codes"], ora["margins"].numpy(), MARGIN, min_exact_rate=0.9,
                              what="config-4 golden")
    if not (res["first_stage"] >= 0).any():
        assert np.abs(r["recon_speech"].cpu().numpy() - z["recon"]).max() <= WAV_TOL
    d = model.inference_decoding_emb(torch.from_numpy(z["quant"]))
    dref = oracle.decode_frame(torch.from_numpy(z["quant"]), None)
    assert (d["recon_speech"].cpu() - dref).abs().max().item() <= WAV_TOL * 10      # un-scaled output (~10x amplitude)


# ---------------------------------------------------------------------------------------------- layer level (2-D)
_STRIDES2 = {"encoder.model.3": (4, 1), "encoder.model.6": (4, 2), "encoder.model.9": (4, 1), "encoder.model.12": (4, 1),
             "decoder.model.4": (4, 1), "decoder.model.7": (4, 1), "decoder.model.10": (4, 2), "decoder.model.13": (4, 1)}
_OUT_PAD = {"decoder.model.13": ((0, 1), (0, 0))}            # SEANetDecoder2d last_out_padding (seanet_decoder.py:262)

CASES2 = [  # (layer, C_in, F, T, elu)
    ("encoder.model.0", 3, 40, 150, False), ("encoder.model.1.block.1", 32, 20, 140, True),
    ("encoder.model.1.block.3", 16, 9, 300, True), ("encoder.model.1.shortcut", 32, 7, 129, False),
    ("encoder.model.3", 32, 37, 131, True), ("encoder.model.4.block.1", 64, 12, 200, True),
    ("encoder.model.6", 64, 16, 201, True), ("encoder.model.9", 128, 16, 130, True),
    ("encoder.model.10.block.1", 256, 4, 150, True), ("encoder.model.12", 256, 4, 140, True),
    ("decoder.model.4", 512, 1, 129, True), ("decoder.model.7", 256, 4, 130, True), ("decoder.model.10", 128, 16, 70, True),
    ("decoder.model.13", 64, 64, 100, True), ("decoder.model.14.block.1", 32, 30, 133, True),
    ("decoder.model.16", 32, 40, 150, True), ("decoder.model.16", 32, 257, 11, True),
]


def _truth2d(sd, layer, x_bcft, elu):
    """float64 raw (pre-GroupNorm) output [B, C, F_raw, T_raw] and the logical window (f_off, t_off, F, T)."""
    from oracle import encodec_oracle as O
    from oracle.freqcodec_oracle import pad2d_reflect
    x = x_bcft.double()
    if elu:
        x = torch.nn.functional.elu(x)
    if layer + ".convtr.convtr.weight" in sd:
        w, b = sd[layer + ".convtr.convtr.weight"].double(), sd[layer + ".convtr.convtr.bias"].double()
        sf, st = _STRIDES2[layer]
        y = torch.nn.functional.conv_transpose2d(x, w, b, stride=(sf, st))
        kf, kt = w.shape[-2:]
        pf, pt = kf - sf, kt - st
        pf_r, pt_r = pf // 2, pt // 2
        pf_l, pt_l = pf - pf_r, pt - pt_r
        (fo_l, fo_r), (to_l, to_r) = _OUT_PAD.get(layer, ((0, 0), (0, 0)))
        tl, tr = max(pt_l - to_l, 0), max(pt_r - to_r, 0)
        fl, fr = max(pf_l - fo_l, 0), max(pf_r - fo_r, 0)
        return y, (fl, tl, y.shape[-2] - fl - fr, y.shape[-1] - tl - tr)
    w, b = sd[layer + ".conv.conv.weight"].double(), sd[layer + ".conv.conv.bias"].double()
    kf, kt = w.shape[-2:]
    sf, st = _STRIDES2.get(layer, (1, 1))
    pt_f, pt_t = (kf - 1) - (sf - 1), (kt - 1) - (st - 1)
    extra_t = O.extra_padding_for_conv1d(x.shape[-1], kt, st, pt_t)
    f_after, t_after = pt_f // 2, pt_t // 2
    y = torch.nn.functional.conv2d(pad2d_reflect(x, (pt_t - t_after + extra_t, t_after), (pt_f - f_after, f_after)), w, b,
                                   stride=(sf, st))
    return y, (0, 0, y.shape[-2], y.shape[-1])


# the small golden model (n_filters 4): C_in 4 / 8 / 16 with several frequency taps per chunk, phase scatter with 4 / 8
# channels per phase, C_out 2 / 4 / 8 padded to the 16-column n-tile
CASES2_SMALL = [
    ("encoder.model.0", 3, 30, 140, False), ("encoder.model.1.block.1", 4, 20, 140, True),
    ("encoder.model.1.shortcut", 4, 7, 129, False), ("encoder.model.3", 4, 37, 131, True),
    ("encoder.model.4.block.1", 8, 12, 200, True), ("encoder.model.4.block.3", 4, 12, 150, True),
    ("encoder.model.6", 8, 16, 201, True), ("encoder.model.7.block.1", 16, 8, 150, True),
    ("encoder.model.9", 16, 16, 130, True), ("decoder.model.7", 32, 4, 130, True), ("decoder.model.10", 16, 16, 70, True),
    ("decoder.model.13", 8, 64, 100, True), ("decoder.model.14.block.1", 4, 30, 133, True),
    ("decoder.model.16", 4, 40, 150, True),
]


def _check_conv2d_layer(model, sd, layer, cin, F, T, elu, tc2d):
    model.set_option("use_tc2d", tc2d)
    try:
        g = torch.Generator().manual_seed(zlib.crc32(f"{layer}/{cin}/{F}/{T}".encode()))     # reproducible across runs
        B = 2
        x = torch.randn(B, F, T, cin, generator=g)
        y, stats, win = model.debug_conv2d(layer, x, elu=elu)
    finally:
        model.set_option("use_tc2d", 7)
    ref, ref_win = _truth2d(sd, layer, x.permute(0, 3, 1, 2), elu)
    ref_bftc = ref.permute(0, 2, 3, 1)
    y = y.cpu().double()
    assert win == ref_win, (win, ref_win)
    assert tuple(y.shape) == tuple(ref_bftc.shape), (y.shape, ref_bftc.shape)
    rms = ref_bftc.pow(2).mean().sqrt().item()
    err = (y - ref_bftc).abs().max().item()
    print(f"use_tc2d={tc2d} C_in={cin:3d} {layer:26s} F={F:3d} T={T:4d} max-abs err {err:.3e} rms {rms:.3e} rel {err / rms:.3e}")
    assert err <= 2e-5 * rms, (tc2d, layer, err, rms)
    st = stats.cpu().double()
    mean = ref.mean(dim=(1, 2, 3))
    rstd = 1.0 / torch.sqrt(ref.var(dim=(1, 2, 3), unbiased=False) + 1e-5)
    assert (st[:, 0] - mean).abs().max().item() <= 1e-5 * rms
    assert ((st[:, 1] - rstd) / rstd).abs().max().item() <= 1e-5


@pytest.mark.parametrize("tc2d", [7, 0])
@pytest.mark.parametrize("layer,cin,F,T,elu", CASES2)
def test_conv2d_layer(layer, cin, F, T, elu, tc2d):
    """Every 2-D conv family of config 4 through fcb_debug_conv2d on both kernels vs a float64 CPU evaluation.
    Bar as in test_gpu_layers.py: max-abs error <= 2e-5 x rms(output), statistics to 1e-5 relative."""
    cfg, sd, model, _ = _full()
    _check_conv2d_layer(model, sd, layer, cin, F, T, elu, tc2d)


@pytest.mark.parametrize("tc2d", [7, 0])
@pytest.mark.parametrize("layer,cin,F,T,elu", CASES2_SMALL)
def test_conv2d_layer_small_channels(golden_dir, layer, cin, F, T, elu, tc2d):
    z, cfg, sd, model, _ = _small(golden_dir)
    _check_conv2d_layer(model, sd, layer, cin, F, T, elu, tc2d)


# ---------------------------------------------------------------------------------------------- alternative kernel paths
def test_output_conv_padded_tile_path(golden_dir):
    """`conv2d_small_cout` = 0: the 32 -> 3 output conv on the padded tensor-core n-tile (class 4) instead of the default
    halo-tile SIMT kernel -- both stay covered."""
    cfg, sd, model, oracle = _full()
    model.set_option("conv2d_small_cout", 0)
    try:
        for layer, cin, F, T, elu in [("decoder.model.16", 32, 40, 150, True), ("decoder.model.16", 32, 257, 11, True),
                                      ("decoder.model.16", 32, 9, 333, False)]:
            _check_conv2d_layer(model, sd, layer, cin, F, T, elu, 7)
    finally:
        model.set_option("conv2d_small_cout", 1)


@pytest.mark.parametrize("stft_tc", [1, 0])
def test_stft_paths(golden_dir, stft_tc):
    """STFT / iSTFT as tensor-core GEMMs (default) and as the direct-DFT kernels (`stft_tc` = 0) against the oracle
    (torch.stft / istft): config-4 architecture and the small golden model, encoder output and decode-only waveform."""
    from parity_utils import record_parity
    for getter in (_full, lambda: _small(golden_dir)[1:]):
        cfg, sd, model, oracle = getter()
        model.set_option("stft_tc", stft_tc)
        try:
            g = torch.Generator().manual_seed(9)
            wav = 0.1 * torch.randn(2, 160 * 33 + 17, generator=g)
            ora = oracle.inference(wav, want_margin=True)
            r = model.inference(wav, need_recon=True, need_encoder_out=True, need_sub_quants=False)
            err = (r["encoder_out"].cpu() - ora["encoder_out"]).abs().max().item()
            quant = ora["code_embeddings"][0][0]
            d = model.inference_decoding_emb(quant)
            dref = oracle.decode_frame(quant, None)
            derr = (d["recon_speech"].cpu() - dref).abs().max().item()
            record_parity(f"stft_tc={stft_tc} {cfg.name}", kind="stft", encoder_out_max_abs=err, decode_only_max_abs_unscaled=derr)
            assert err <= EMB_TOL
            assert derr <= WAV_TOL * 10                  # un-scaled output (~10x amplitude)
        finally:
            model.set_option("stft_tc", 1)


def _golden_model_check(golden_dir, fname, what, min_exact_rate=0.9):
    from funcodec_b200.encodec import B200Encodec
    from parity_utils import record_parity
    z = np.load(os.path.join(golden_dir, fname))
    cfg = get_config(str(z["cfg_name"]))
    sd = init_state_dict(cfg, int(z["seed"]))
    model = B200Encodec(cfg, sd, "cuda:0")
    wav = torch.from_numpy(z["wav"])
    oracle = OracleFreqCodec(sd, list(zip(cfg.ratios_f, cfg.ratios)))
    ora = oracle.inference(wav, want_margin=True)
    r = model.inference(wav, need_recon=True, need_encoder_out=True, need_sub_quants=False)
    enc_err = np.abs(r["encoder_out"].cpu().numpy() - z["encoder_out"]).max()
    assert enc_err <= EMB_TOL, enc_err
    res = assert_codes_parity(r["code_indices"][0].cpu().numpy(), z["codes"], ora["margins"].numpy(), MARGIN,
                              min_exact_rate=min_exact_rate, what=what, encoder_out_max_abs=float(enc_err))
    assert tuple(r["recon_speech"].shape) == tuple(z["recon"].shape)
    ok_clip = ~(res["first_stage"] >= 0).any(axis=1)
    recon = r["recon_speech"].cpu().numpy()
    werr = 0.0
    for b in np.nonzero(ok_clip)[0]:
        werr = max(werr, float(np.abs(recon[b] - z["recon"][b]).max()))
    # decode-only (no flips involved): the reference's own quantized embeddings through the decoder
    d = model.inference_decoding_emb(torch.from_numpy(z["quant"]))
    dref = oracle.decode_frame(torch.from_numpy(z["quant"]), None)
    derr = (d["recon_speech"].cpu() - dref).abs().max().item()
    record_parity(what, kind="waveform", clips_without_flips=int(ok_clip.sum()), clips=int(ok_clip.size), recon_max_abs=werr,
                  decode_only_max_abs_unscaled=derr)
    assert werr <= WAV_TOL, werr
    assert derr <= WAV_TOL * 10
    return model, cfg


def test_grouped_freq_model(golden_dir):
    """conv_group_ratio / tr_conv_group_ratio > 0 on the small model against vectors of the unmodified grouped reference."""
    _golden_model_check(golden_dir, "freq_magphase_small_grouped.npz", "freq grouped small golden")


def test_config4_gr8_arch_golden(golden_dir):
    """BASELINE config 4 AS NAMED (gr8: conv_group_ratio = tr_conv_group_ratio = 8, full widths) against vectors of the
    unmodified grouped reference FreqCodec (tools/gen_golden_freq_gr8.py)."""
    _golden_model_check(golden_dir, "freq_magphase_config4_gr8_arch.npz", "config-4 gr8 golden")


def test_freq_ds640_ratio_set(golden_dir):
    """conf/freqcodec_mag_phase_16k_n32_600k_step_ds640.yaml's ratio set (time strides 2, 1, 2, 1) against the reference."""
    _golden_model_check(golden_dir, "freq_magphase_small_ds640.npz", "freq ds640 ratio set golden")
