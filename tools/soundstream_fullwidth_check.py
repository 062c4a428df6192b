"""The SoundStream YAMLs at their own widths (n_filters 32, D = 512, three dilated residual blocks per stage, no sequence model)
-- conf/soundstream_noncausal_16k_n32_600k_step.yaml (time_group_norm) and conf/soundstream_16k_n32_600k_step.yaml (weight_norm,
causal) -- against the CPU oracle on both conv paths, one line per case:  python tools/soundstream_fullwidth_check.py

The same comparison lives in tests/test_gpu_fullshape.py::test_soundstream_yaml_widths.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from funcodec_b200 import get_config, init_state_dict  # noqa: E402
from funcodec_b200.encodec import B200Encodec  # noqa: E402
from oracle import encodec_oracle as O  # noqa: E402
from parity_utils import classify_codes  # noqa: E402

MARGIN = 4e-3      # D = 512: the fp32 rounding noise of a distance grows like sqrt(D): the D = 128 margin (2e-3) x 2
WAV_TOL = 1e-4


def main():
    bad = 0
    cases = {}
    for name in ("soundstream_noncausal_16k_n32_ds320", "soundstream_16k_n32_ds320"):
        cfg = get_config(name)
        sd = init_state_dict(cfg, 0)
        wav = 0.1 * torch.randn(2, 48000, generator=torch.Generator().manual_seed(6006))
        oracle = O.OracleEncodec.from_config(sd, cfg)
        ora = oracle.inference(wav, want_margin=True)
        # decode-only reference: the oracle's own quantized embeddings through ITS decoder (no scale applied on this path)
        ora["decode_emb"] = oracle.inference_decoding_emb(ora["code_embeddings"][0][0])["recon_speech"]
        cases[name] = (cfg, sd, wav, ora)
    for use_tc in (1, 0):
        for name, (cfg, sd, wav, ora) in cases.items():
            model = B200Encodec(cfg, sd, "cuda:0", options={"use_tc": use_tc})
            r = model.inference(wav, need_recon=True, need_encoder_out=True, need_sub_quants=False)
            enc_err = float((r["encoder_out"].cpu() - ora["encoder_out"]).abs().max())
            codes = r["code_indices"][0].cpu().numpy()
            res = classify_codes(codes, ora["code_indices"][0].numpy(), ora["margins"].numpy(), MARGIN)
            ok_clip = ~(res["first_stage"] >= 0).any(axis=1)
            rec, ref = r["recon_speech"].cpu(), ora["recon_speech"]
            werr = max([float((rec[b] - ref[b]).abs().max()) for b in np.nonzero(ok_clip)[0]] or [0.0])
            # decode-only: the oracle's own quantized embeddings in (no index contamination)
            d = model.inference_decoding_emb(ora["code_embeddings"][0][0])
            derr = float((d["recon_speech"].cpu() - ora["decode_emb"]).abs().max())
            frames = codes.shape[1] * codes.shape[2]
            ok = res["bad_frames"] == 0 and res["near_tie_frames"] <= max(2, frames // 100) and werr <= WAV_TOL and derr <= WAV_TOL
            bad += not ok
            print(f"{'OK ' if ok else 'FAIL'} {name} use_tc={use_tc}: encoder_out max-abs {enc_err:.2e}, frames {frames}, "
                  f"near-tie flips {res['near_tie_frames']}, bad {res['bad_frames']}, worst accepted margin {res['worst_margin']:.2e}, "
                  f"recon max-abs {werr:.2e}, decode-only {derr:.2e}", flush=True)
            del model
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
