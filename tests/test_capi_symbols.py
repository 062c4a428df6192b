"""The C-ABI library loads on a CPU-only box and exports every symbol include/funcodec_b200.h declares
(no compute calls without a GPU); host-side config logic matches the reference formulas."""
import ctypes
import os
import re

import pytest

from funcodec_b200 import _capi, get_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "funcodec_b200.h")).read()
    declared = set(re.findall(r"FCB_API\s+[\w\s\*]+?\b(fcb_\w+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(_capi.SYMBOLS), (declared ^ set(_capi.SYMBOLS))
    lib = _capi.load_library()
    for name in declared:
        assert hasattr(lib, name)
    assert lib.fcb_version().startswith(b"funcodec_b200")


def test_create_without_gpu_fails_loudly_not_silently():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from funcodec_b200.encodec import B200Encodec
    from funcodec_b200 import init_state_dict
    cfg = get_config("tiny_ds40")
    with pytest.raises(Exception):
        B200Encodec(cfg, init_state_dict(cfg, 0), "cuda:0")
    with pytest.raises(_capi.FcbError):
        B200Encodec(cfg, init_state_dict(cfg, 0), "cpu")


def test_bandwidth_to_quantizers():
    """vq.py:105-117 and codec_inference.py:121-125."""
    cfg = get_config("encodec_16k_n32_ds640")
    assert cfg.bandwidth_per_quantizer() == 250.0
    assert [cfg.num_quantizers_for_bandwidth(b) for b in (None, 0, 250, 499, 4000, 8000, 99999)] == [32, 32, 1, 1, 16, 32, 399]
    cfg = get_config("encodec_16k_n32_ds320")
    assert cfg.bandwidth_per_quantizer() == 500.0 and cfg.hop_length == 320 and cfg.frames(480000) == 1500


def test_config_from_reference_like_model():
    """integration.config_from_reference_model on a duck-typed stand-in for the reference Encodec module."""
    import types
    import torch
    from funcodec_b200 import init_state_dict
    from funcodec_b200.integration import config_from_reference_model, UnsupportedReferenceModel
    cfg = get_config("encodec_16k_n32_ds320")
    sd = init_state_dict(cfg, 0)
    m = types.SimpleNamespace(
        encoder=types.SimpleNamespace(ratios=list(reversed(cfg.ratios))), decoder=types.SimpleNamespace(ratios=list(cfg.ratios)),
        quantizer=types.SimpleNamespace(sampling_rate=16000, encoder_hop_length=320, codebook_size=1024, input_proj=None, input_act=None),
        audio_normalize=True, segment_dur=None, codec_domain="time", state_dict=lambda: sd)
    got = config_from_reference_model(m)
    for f in ("ratios", "n_filters", "dimension", "kernel_size", "last_kernel_size", "residual_kernel_size", "lstm_layers",
              "codebook_size", "num_quantizers", "sample_rate", "audio_normalize"):
        assert getattr(got, f) == getattr(cfg, f), f
    m.segment_dur = 1.0                     # segmenting is handled by the wrapper (fcb_roundtrip_segmented), not the config
    assert config_from_reference_model(m).ratios == cfg.ratios
    m.quantizer.input_proj = object()
    with pytest.raises(UnsupportedReferenceModel):
        config_from_reference_model(m)


def test_config_from_reference_like_freqcodec():
    """Same, for a mag_phase FreqCodec (codec_freq.py:118-215): [freq, time] ratio pairs, domain_conf."""
    import types
    from funcodec_b200 import init_state_dict
    from funcodec_b200.integration import config_from_reference_model, UnsupportedReferenceModel
    cfg = get_config("freq_small")
    sd = init_state_dict(cfg, 0)
    pairs = [[f, t] for f, t in zip(cfg.ratios_f, cfg.ratios)]
    m = types.SimpleNamespace(
        encoder=types.SimpleNamespace(ratios=list(reversed(pairs))), decoder=types.SimpleNamespace(ratios=pairs),
        quantizer=types.SimpleNamespace(sampling_rate=cfg.sample_rate, encoder_hop_length=cfg.hop_length,
                                        codebook_size=cfg.codebook_size, input_proj=None, input_act=None),
        audio_normalize=True, segment_dur=None, codec_domain=["mag_phase", "mag_phase"],
        domain_conf={"n_fft": cfg.n_fft, "hop_length": cfg.stft_hop}, state_dict=lambda: sd)
    got = config_from_reference_model(m)
    for f in ("arch", "ratios", "ratios_f", "n_fft", "stft_hop", "n_filters", "dimension", "kernel_size", "last_kernel_size",
              "residual_kernel_size", "lstm_layers", "codebook_size", "num_quantizers"):
        assert getattr(got, f) == getattr(cfg, f), f
    assert (got.conv_group_ratio, got.tr_conv_group_ratio) == (-1, -1)
    # grouped 2-D convs: the ratios are recovered from the weight shapes
    gcfg = get_config("freq_small_grouped")
    gsd = init_state_dict(gcfg, 0)
    m.state_dict = lambda: gsd
    got = config_from_reference_model(m)
    assert (got.conv_group_ratio, got.tr_conv_group_ratio, got.n_filters) == (gcfg.conv_group_ratio, gcfg.tr_conv_group_ratio, gcfg.n_filters)
    m.state_dict = lambda: sd
    m.segment_dur = 1.0
    with pytest.raises(UnsupportedReferenceModel):
        config_from_reference_model(m)
    m.segment_dur = None
    m.codec_domain = ["stft", "stft"]
    with pytest.raises(UnsupportedReferenceModel):
        config_from_reference_model(m)


REF_MODULES = os.path.join(ROOT, "tests", "golden", "reference_modules.json")


def _reference_models():
    """The reference `Encodec` objects as recorded from the unmodified reference by tools/gen_golden_reference_modules.py:
    module tree (class names, option attributes, children) and state_dict key -> shape map per preset."""
    import json
    with open(REF_MODULES) as f:
        return json.load(f)


class _RefModule:
    """Stand-in for one recorded reference module: same class name, recorded attributes, children by name (and by index
    for Sequential / ModuleList), modules() in registration order like nn.Module."""

    def __init__(self, rec):
        self._children = {}
        for k, v in rec["attrs"].items():
            setattr(self, k, tuple(v) if k == "dilation" else v)
        for name, child in rec["children"]:
            self._children[name] = _rebuild(child)

    def __getattr__(self, k):
        ch = self.__dict__.get("_children", {})
        if k in ch:
            return ch[k]
        raise AttributeError(k)

    def __getitem__(self, i):
        return self._children[str(i)]

    def modules(self):
        yield self
        for c in self._children.values():
            yield from c.modules()


def _rebuild(rec):
    import torch.nn as nn
    if rec["type"] == "ELU":                 # isinstance checks in integration._check_module_options
        return nn.ELU(alpha=rec["attrs"]["alpha"])
    if rec["type"] == "GroupNorm":
        return nn.GroupNorm(rec["attrs"]["num_groups"], rec["attrs"]["num_channels"])
    return type(rec["type"], (_RefModule,), {})(rec)


def _reference_encodec(rec):
    import torch
    m = _rebuild(rec["tree"])
    sd = {k: torch.empty(shp, device="meta") for k, shp in rec["state_dict"].items()}
    m.state_dict = lambda: sd
    return m


def test_config_from_the_real_reference_modules():
    """integration.config_from_reference_model + state_dict name coverage on the REAL reference `Encodec` (ds320, tiny_ds40,
    the SoundStream / weight_norm variants; recorded from the unmodified reference in tests/golden/reference_modules.json):
    every field matches the preset, every tensor the engine needs is in the reference's state_dict under the same name and
    shape, and option variants that keep the shapes are refused."""
    from funcodec_b200.integration import config_from_reference_model, stacked_codebooks, UnsupportedReferenceModel
    from funcodec_b200.weights import state_dict_shapes
    models = _reference_models()["models"]
    names = ("encodec_16k_n32_ds320", "tiny_ds40", "soundstream_noncausal_small", "soundstream_causal_small", "weightnorm_lstm_small")
    assert set(names) <= set(models)
    for name in names:
        cfg = get_config(name)
        m = _reference_encodec(models[name])
        got = config_from_reference_model(m)
        for f in ("arch", "ratios", "n_filters", "dimension", "kernel_size", "last_kernel_size", "residual_kernel_size",
                  "lstm_layers", "codebook_size", "num_quantizers", "sample_rate", "audio_normalize", "n_residual_layers",
                  "dilation_base", "norm", "causal"):
            assert getattr(got, f) == getattr(cfg, f), (name, f)
        sd = m.state_dict()
        for k, shp in state_dict_shapes(cfg).items():
            assert k in sd and tuple(sd[k].shape) == tuple(shp), (name, k)
        assert tuple(stacked_codebooks(sd).shape) == (cfg.num_quantizers, cfg.codebook_size, cfg.dimension)
    # options that keep parameter names and shapes but change the maths are refused
    m = _reference_encodec(models["tiny_ds40"])
    m.encoder.model[0].causal = True                   # one causal conv among non-causal ones / causal under GroupNorm
    with pytest.raises(UnsupportedReferenceModel):
        config_from_reference_model(m)
    m.encoder.model[0].causal = False
    m.decoder.model[0].pad_mode = "constant"
    with pytest.raises(UnsupportedReferenceModel):
        config_from_reference_model(m)
    m.decoder.model[0].pad_mode = "reflect"
    m.quantizer.rq.model.q0_ds_ratio = 2
    with pytest.raises(UnsupportedReferenceModel):
        config_from_reference_model(m)


def test_use_ddp_false_reference_quantizer_keys():
    """`use_ddp: false` (core_vq.py:147-150): the reference's own per-layer key names (recorded from the unmodified
    reference's ResidualVectorQuantization in tests/golden/reference_modules.json) are what stacked_codebooks /
    fcb_finalize assemble into the [n_q, K, D] codebook tensor."""
    import torch
    from funcodec_b200.integration import stacked_codebooks
    rec = _reference_models()["use_ddp_false_rvq"]
    n_q, D, K = rec["num_quantizers"], rec["dim"], rec["codebook_size"]
    # the RVQ class sits at quantizer.rq.model
    sd = {"quantizer.rq.model." + k: torch.zeros(shp) for k, shp in rec["state_dict"].items()}
    assert "quantizer.rq.model.layers.0._codebook.embed" in sd and "quantizer.rq.model.embed" not in sd
    for i in range(n_q):
        assert tuple(sd[f"quantizer.rq.model.layers.{i}._codebook.embed"].shape) == (K, D)
        sd[f"quantizer.rq.model.layers.{i}._codebook.embed"] = torch.full((K, D), float(i))
    e = stacked_codebooks(sd)
    assert tuple(e.shape) == (n_q, K, D) and [float(e[i, 0, 0]) for i in range(n_q)] == [0.0, 1.0, 2.0]
