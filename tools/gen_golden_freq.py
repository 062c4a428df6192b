"""Golden vectors for the FreqCodec (mag_phase) path from the UNMODIFIED reference (build container only).
Weights: funcodec_b200.weights.init_state_dict(cfg, seed) loaded into the reference modules; the fixtures store the seed and a
checksum of the weights, not the weights themselves."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from ref_harness import import_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


def build(n_filters, dimension, K, nq, ratios, conv_group_ratio=-1, tr_conv_group_ratio=-1, hop=320):
    import_reference()
    from funcodec.models import codec_freq
    codec_freq.check_argument_types = lambda: True
    from funcodec.models.encoder.seanet_encoder import SEANetEncoder2d
    from funcodec.models.decoder.seanet_decoder import SEANetDecoder2d
    from funcodec.models.quantizer.costume_quantizer import CostumeQuantizer
    torch.manual_seed(5)
    enc = SEANetEncoder2d(input_size=3, dimension=dimension, n_filters=n_filters, ratios=ratios, norm="time_group_norm",
                          norm_params={"num_groups": 1}, causal=False, dilation_base=1, conv_group_ratio=conv_group_ratio)
    dec = SEANetDecoder2d(input_size=dimension, channels=3, n_filters=n_filters, ratios=ratios, norm="time_group_norm",
                          norm_params={"num_groups": 1}, causal=False, dilation_base=1, conv_group_ratio=conv_group_ratio,
                          tr_conv_group_ratio=tr_conv_group_ratio)
    q = CostumeQuantizer(input_size=dimension, codebook_size=K, num_quantizers=nq, kmeans_init=False, sampling_rate=16000,
                         encoder_hop_length=hop, use_ddp=True)
    m = codec_freq.FreqCodec(input_size=3, odim=dimension, encoder=enc, quantizer=q, decoder=dec, discriminator=None,
                             target_sample_hz=16000, multi_spectral_window_powers_of_two=[], audio_normalize=True,
                             segment_dur=None, overlap_ratio=None, codec_domain=["mag_phase", "mag_phase"])
    g = torch.Generator().manual_seed(6)
    with torch.no_grad():
        for name, par in m.named_parameters():
            if name.endswith("norm.weight"):
                par.copy_(1 + 0.1 * torch.randn(par.shape, generator=g))
            elif name.endswith("norm.bias"):
                par.copy_(0.1 * torch.randn(par.shape, generator=g))
        m.quantizer.rq.model.embed.copy_(torch.randn(nq, K, dimension, generator=g) * (0.6 * 0.9 ** torch.arange(nq).float()).view(nq, 1, 1))
        m.quantizer.rq.model.inited.fill_(1)
    return m.eval()


if __name__ == "__main__":
    torch.set_num_threads(8)
    from funcodec_b200 import get_config, init_state_dict
    ratios = [[4, 1], [4, 1], [4, 2], [4, 1]]
    cfg = get_config("freq_small")
    sd = init_state_dict(cfg, 0)
    m = build(cfg.n_filters, cfg.dimension, cfg.codebook_size, cfg.num_quantizers, ratios)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.split(".")[-1] in ("cluster_size", "embed_avg", "inited", "window") for k in missing), (missing, unexpected)
    m.quantizer.rq.model.inited.fill_(1)
    g = torch.Generator().manual_seed(8)
    wav = 0.1 * torch.randn(2, 3200 + 57, generator=g)
    with torch.no_grad():
        r = m.inference(wav, need_recon=True, bit_width=None, use_scale=True)
        emb, scale = m._encode(wav.unsqueeze(1))[0]
    out = dict(cfg_name=cfg.name, seed=0, wav=wav.numpy(), ratios=np.array(ratios), codes=r["code_indices"][0].numpy().astype(np.int16),
               quant=r["code_embeddings"][0][0].numpy(), scale=r["code_embeddings"][0][1].numpy(),
               recon=r["recon_speech"].numpy(), encoder_out=emb.numpy(),
               sd_checksum=float(sum(v.double().abs().sum().item() for v in sd.values())))
    path = os.path.join(OUT, "freq_magphase_small.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB", "codes", out["codes"].shape, "recon", out["recon"].shape)

    # BASELINE config 4 architecture (repo YAML: n_filters 32, D 128, K 1024, n_q 32, groups = 1) on a short clip; weights
    # are funcodec_b200.weights.init_state_dict(cfg, 0) loaded into the reference module (not stored in the fixture)
    cfg = get_config("freqcodec_magphase_16k_n32_ds320")
    sd = init_state_dict(cfg, 0)
    m = build(cfg.n_filters, cfg.dimension, cfg.codebook_size, cfg.num_quantizers, ratios)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.split(".")[-1] in ("cluster_size", "embed_avg", "inited", "window") or "discriminator" in k for k in missing), (missing, unexpected)
    m.quantizer.rq.model.inited.fill_(1)
    g = torch.Generator().manual_seed(4)
    wav = 0.1 * torch.randn(1, 8000, generator=g)
    with torch.no_grad():
        r = m.inference(wav, need_recon=True, bit_width=None, use_scale=True)
        emb, scale = m._encode(wav.unsqueeze(1))[0]
    out = dict(cfg_name=cfg.name, seed=0, wav=wav.numpy(), codes=r["code_indices"][0].numpy().astype(np.int16),
               quant=r["code_embeddings"][0][0].numpy(), scale=r["code_embeddings"][0][1].numpy(), recon=r["recon_speech"].numpy(),
               encoder_out=emb.numpy(), sd_checksum=float(sum(v.double().abs().sum().item() for v in sd.values())))
    path = os.path.join(OUT, "freq_magphase_config4_arch.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB", "codes", out["codes"].shape, "recon", out["recon"].shape)

    # grouped 2-D convs (conv_group_ratio / tr_conv_group_ratio > 0): a small model, weights = init_state_dict(cfg, 0)
    cfg = get_config("freq_small_grouped")
    sd = init_state_dict(cfg, 0)
    m = build(cfg.n_filters, cfg.dimension, cfg.codebook_size, cfg.num_quantizers, ratios, cfg.conv_group_ratio, cfg.tr_conv_group_ratio)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.split(".")[-1] in ("cluster_size", "embed_avg", "inited", "window") for k in missing), (missing, unexpected)
    m.quantizer.rq.model.inited.fill_(1)
    g = torch.Generator().manual_seed(9)
    wav = 0.1 * torch.randn(2, 3200 + 31, generator=g)
    with torch.no_grad():
        r = m.inference(wav, need_recon=True, bit_width=None, use_scale=True)
        emb, scale = m._encode(wav.unsqueeze(1))[0]
    out = dict(cfg_name=cfg.name, seed=0, wav=wav.numpy(), codes=r["code_indices"][0].numpy().astype(np.int16),
               quant=r["code_embeddings"][0][0].numpy(), scale=r["code_embeddings"][0][1].numpy(), recon=r["recon_speech"].numpy(),
               encoder_out=emb.numpy(), sd_checksum=float(sum(v.double().abs().sum().item() for v in sd.values())))
    path = os.path.join(OUT, "freq_magphase_small_grouped.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB", "codes", out["codes"].shape, "recon", out["recon"].shape)

    # the ds640 ratio set of conf/freqcodec_mag_phase_16k_n32_600k_step_ds640.yaml (time strides 2, 1, 2, 1), small widths
    cfg = get_config("freq_small_ds640")
    sd = init_state_dict(cfg, 0)
    ratios640 = [[f, t] for f, t in zip(cfg.ratios_f, cfg.ratios)]
    m = build(cfg.n_filters, cfg.dimension, cfg.codebook_size, cfg.num_quantizers, ratios640, hop=640)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.split(".")[-1] in ("cluster_size", "embed_avg", "inited", "window") for k in missing), (missing, unexpected)
    m.quantizer.rq.model.inited.fill_(1)
    g = torch.Generator().manual_seed(10)
    wav = 0.1 * torch.randn(2, 6400 + 333, generator=g)
    with torch.no_grad():
        r = m.inference(wav, need_recon=True, bit_width=None, use_scale=True)
        emb, scale = m._encode(wav.unsqueeze(1))[0]
    out = dict(cfg_name=cfg.name, seed=0, wav=wav.numpy(), codes=r["code_indices"][0].numpy().astype(np.int16),
               quant=r["code_embeddings"][0][0].numpy(), scale=r["code_embeddings"][0][1].numpy(), recon=r["recon_speech"].numpy(),
               encoder_out=emb.numpy(), sd_checksum=float(sum(v.double().abs().sum().item() for v in sd.values())))
    path = os.path.join(OUT, "freq_magphase_small_ds640.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB", "codes", out["codes"].shape, "recon", out["recon"].shape)
