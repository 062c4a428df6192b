"""Full-shape parity on every BASELINE.json config (the shapes the bench is quoted on), through the C ABI, against the CPU oracle.
Every comparison is recorded (parity_utils.RECORDS -> parity_records.json): frames, exact
frames, near-tie frames, worst accepted oracle margin, waveform max-abs on clips whose codes all match, batch-consistency.

  config 1/2  ds640, 10 s: B = 16, ALL clips against the oracle (B = 1 = config 1 is clip 0 run alone)
  config 3    ds320, one 30 s clip (T' = 1500 LSTM steps, the longest recurrence in the suite) at n_q = 32; the n_q sweep
              {2,4,8,16,32} is the prefix property; + the B = 64 shape (finite, deterministic, batch-consistent with the 1-clip run)
  config 4    FreqCodec mag_phase ds320, B = 2 x 10 s, groups = 1 and gr8 (as named)
  config 5    ds640, B = 64 per GPU (8 LSTM clip groups at H = 1024): 2 clips against the oracle + consistency with B = 16
  (f) N2      the SoundStream YAMLs at their real widths (n_filters 32, D = 512 -> column-sliced fp32 RVQ kernel, 3 dilated residual
              blocks per stage, no sequence model): non-causal time_group_norm and causal weight_norm, B = 2 x 3 s
"""
import numpy as np
import pytest
import torch

from funcodec_b200 import get_config, init_state_dict
from oracle import encodec_oracle as O
from oracle.freqcodec_oracle import OracleFreqCodec
from parity_utils import assert_codes_parity, record_parity

pytestmark = pytest.mark.gpu

WAV_TOL = 1e-4
MARGIN = 2e-3
_M = {}


def _time_model(name):
    from funcodec_b200.encodec import B200Encodec
    if name not in _M:
        cfg = get_config(name)
        sd = init_state_dict(cfg, 0)
        _M[name] = (cfg, sd, B200Encodec(cfg, sd, "cuda:0"), O.OracleEncodec.from_config(sd, cfg))
    return _M[name]


def _freq_model(name):
    from funcodec_b200.encodec import B200Encodec
    if name not in _M:
        cfg = get_config(name)
        sd = init_state_dict(cfg, 0)
        _M[name] = (cfg, sd, B200Encodec(cfg, sd, "cuda:0"),
                    OracleFreqCodec(sd, list(zip(cfg.ratios_f, cfg.ratios)), cfg.sample_rate, cfg.lstm_layers, cfg.n_fft, cfg.stft_hop))
    return _M[name]


def _compare(what, r, ora, min_exact, scaled=True, clips=None, margin=MARGIN):
    codes = r["code_indices"][0].cpu()
    if clips is not None:
        codes = codes[:, clips]
    res = assert_codes_parity(codes.numpy(), ora["code_indices"][0].numpy(), ora["margins"].numpy(), margin,
                              min_exact_rate=min_exact, what=what)
    ok_clip = ~(res["first_stage"] >= 0).any(axis=1)
    rec = r["recon_speech"].cpu()
    if clips is not None:
        rec = rec[clips]
    ref = ora["recon_speech"]
    n = min(rec.shape[-1], ref.shape[-1])
    werr = max([float((rec[b, ..., :n] - ref[b, ..., :n]).abs().max()) for b in np.nonzero(ok_clip)[0]] or [0.0])
    record_parity(what, kind="waveform", clips=int(ok_clip.size), clips_without_flips=int(ok_clip.sum()), recon_max_abs=werr,
                  tol=WAV_TOL if scaled else 10 * WAV_TOL)
    assert werr <= (WAV_TOL if scaled else 10 * WAV_TOL), werr
    return res


def test_config2_all_16_clips_and_config1():
    cfg, sd, model, oracle = _time_model("encodec_16k_n32_ds640")
    B, L = 16, 160000
    wav = 0.1 * torch.randn(B, L, generator=torch.Generator().manual_seed(2002))
    r = model.inference(wav, need_recon=True, need_sub_quants=False)
    ora = oracle.inference(wav, want_margin=True)
    _compare("config 2: ds640 B=16 x 10 s, n_q=32, all clips", r, ora, 0.99)
    # config 1: one clip alone == the same clip inside the batch up to near-ties (clips never interact)
    r1 = model.inference(wav[:1], need_recon=True, need_sub_quants=False)
    o1 = {k: ([v[0][:, :1]] if k == "code_indices" else v) for k, v in ora.items()}
    o1["margins"] = ora["margins"][:, :1]
    o1["recon_speech"] = ora["recon_speech"][:1]
    _compare("config 1: ds640 B=1 x 10 s, n_q=32", r1, o1, 0.98)
    same = (r1["code_indices"][0][:, 0] == r["code_indices"][0][:, 0]).all(dim=0).float().mean().item()
    record_parity("config 1 vs config 2 (clip 0 alone vs in the batch)", kind="batch_consistency", frame_equal_rate=same)
    assert same >= 0.98


def test_config3_30s_clip_and_bitrate_sweep():
    cfg, sd, model, oracle = _time_model("encodec_16k_n32_ds320")
    L = 480000
    g = torch.Generator().manual_seed(3003)
    wav1 = 0.1 * torch.randn(1, L, generator=g)
    r = model.inference(wav1, need_recon=True, need_sub_quants=False)
    assert tuple(r["code_indices"][0].shape) == (32, 1, 1500)
    ora = oracle.inference(wav1, want_margin=True)
    _compare("config 3: ds320 1 x 30 s (T'=1500), n_q=32", r, ora, 0.98)
    # bitrate sweep n_q in {2,4,8,16,32}: fewer quantizers == prefix of the code matrix, and the oracle agrees on the waveform
    for n_q in (2, 4, 8, 16):
        bw = n_q * cfg.bandwidth_per_quantizer()
        rq = model.inference(wav1, need_recon=True, bit_width=bw, need_sub_quants=False)
        assert torch.equal(rq["code_indices"][0], r["code_indices"][0][:n_q])
        oq = oracle.inference(wav1, bit_width=bw, want_margin=True)
        _compare(f"config 3: ds320 1 x 30 s, n_q={n_q}", rq, oq, 0.98)
    # the B = 64 shape of the config: finite, deterministic, clip 0 consistent with its single-clip run
    B = 64
    wav = torch.cat([wav1, 0.1 * torch.randn(B - 1, L, generator=g)], dim=0)
    rb = model.inference(wav, need_recon=True, need_sub_quants=False)
    rb2 = model.inference(wav, need_recon=True, need_sub_quants=False)
    assert torch.equal(rb["code_indices"][0], rb2["code_indices"][0]) and torch.equal(rb["recon_speech"], rb2["recon_speech"])
    assert torch.isfinite(rb["recon_speech"]).all()
    same = (rb["code_indices"][0][:, 0] == r["code_indices"][0][:, 0]).all(dim=0).float().mean().item()
    record_parity("config 3: clip 0 in the B=64 batch vs alone", kind="batch_consistency", frame_equal_rate=same)
    assert same >= 0.98
    _compare("config 3: ds320 B=64 x 30 s, clip 0 against the oracle", rb, ora, 0.98, clips=[0])


@pytest.mark.parametrize("name,tag", [("freqcodec_magphase_16k_n32_ds320", "groups=1 (repo YAML)"),
                                      ("freqcodec_magphase_16k_n32_ds320_gr8", "gr8 (as named)")])
def test_config4_two_10s_clips(name, tag):
    cfg, sd, model, oracle = _freq_model(name)
    B, L = 2, 160000
    wav = 0.1 * torch.randn(B, L, generator=torch.Generator().manual_seed(4004))
    r = model.inference(wav, need_recon=True, need_sub_quants=False)
    ora = oracle.inference(wav, want_margin=True)
    assert tuple(r["code_indices"][0].shape) == tuple(ora["code_indices"][0].shape) == (32, B, cfg.frames(L))
    _compare(f"config 4: FreqCodec mag_phase ds320 {tag}, B=2 x 10 s, n_q=32", r, ora, 0.95)


def test_config5_b64_per_gpu():
    cfg, sd, model, oracle = _time_model("encodec_16k_n32_ds640")
    B, L = 64, 160000
    wav = 0.1 * torch.randn(B, L, generator=torch.Generator().manual_seed(5005))
    r = model.inference(wav, need_recon=True, need_sub_quants=False)
    assert torch.isfinite(r["recon_speech"]).all()
    sub = [5, 60]
    ora = oracle.inference(wav[sub], want_margin=True)
    _compare("config 5: ds640 B=64/GPU x 10 s, clips 5 and 60 against the oracle", r, ora, 0.98, clips=sub)
    r16 = model.inference(wav[:16], need_recon=True, need_sub_quants=False)
    same = (r16["code_indices"][0] == r["code_indices"][0][:, :16]).all(dim=0).float().mean().item()
    record_parity("config 5: first 16 clips in the B=64 batch vs as a B=16 batch", kind="batch_consistency", frame_equal_rate=same)
    assert same >= 0.98


@pytest.mark.parametrize("name", ["soundstream_noncausal_16k_n32_ds320", "soundstream_16k_n32_ds320"])
def test_soundstream_yaml_widths(name):
    """conf/soundstream_noncausal_16k_n32_600k_step.yaml and conf/soundstream_16k_n32_600k_step.yaml (weight_norm, causal) at the
    YAMLs' own widths against the oracle (which is pinned on the reference for both branches at small widths).  First measured by
    tools/soundstream_fullwidth_check.py."""
    cfg, sd, model, oracle = _time_model(name)
    B, L = 2, 48000
    wav = 0.1 * torch.randn(B, L, generator=torch.Generator().manual_seed(6006))
    r = model.inference(wav, need_recon=True, need_sub_quants=False)
    ora = oracle.inference(wav, want_margin=True)
    assert tuple(r["code_indices"][0].shape) == tuple(ora["code_indices"][0].shape) == (32, B, 150)
    # D = 512: the fp32 rounding noise of a distance grows like sqrt(D), so the near-tie margin is the D = 128 one x 2
    _compare(f"N2 {name}: B=2 x 3 s, n_q=32", r, ora, 0.97, margin=2 * MARGIN)
