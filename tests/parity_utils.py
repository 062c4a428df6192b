"""Shared helpers for the parity tests: margin-classified comparison of RVQ code indices.

SURVEY.md §8(c): bit-exact indices are not attainable unconditionally -- top-2 distance gaps reach one
fp32 ulp of the distance -- so a mismatch is accepted only when the ORACLE's own top-2 margin at the
first diverging stage of that frame is below `margin_tol`; later stages of the frame are excluded
(the residual differs after a flip).
"""
import json
import os

import numpy as np

# Every comparison a test makes is also RECORDED (tests/conftest.py dumps the list at session end to
# parity_records.json, one record per comparison).
RECORDS = []


def record_parity(what, **fields):
    """Append one measured parity record (plain numbers only) -- frames / exact / near-tie counts, worst accepted margin,
    waveform max-abs error ... -- so that the bars asserted in the tests can be compared with what was measured."""
    rec = dict(what=str(what))
    for k, v in fields.items():
        if isinstance(v, (np.floating, np.integer)):
            v = v.item()
        rec[k] = v
    RECORDS.append(rec)
    return rec


def dump_records(path):
    if not RECORDS:
        return
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        json.dump(RECORDS, f, indent=1)


def classify_codes(codes_test, codes_ref, margins_ref, margin_tol):
    """codes_*: [n_q, B, T] ints; margins_ref: [n_q, B, T] oracle (top1 - top2) of -dist.
    Returns dict(exact_frames, total_frames, near_tie_frames, bad_frames, worst_margin)."""
    ct = np.asarray(codes_test).astype(np.int64)
    cr = np.asarray(codes_ref).astype(np.int64)
    mg = np.asarray(margins_ref)
    assert ct.shape == cr.shape == mg.shape, (ct.shape, cr.shape, mg.shape)
    n_q, B, T = ct.shape
    diff = ct != cr
    any_diff = diff.any(axis=0)
    first = np.where(any_diff, diff.argmax(axis=0), -1)       # first diverging stage per frame
    total = B * T
    exact = int((~any_diff).sum())
    near, bad, worst = 0, 0, 0.0
    for b, t in zip(*np.nonzero(any_diff)):
        m = float(mg[first[b, t], b, t])
        worst = max(worst, m)
        if m <= margin_tol:
            near += 1
        else:
            bad += 1
    return dict(exact_frames=exact, total_frames=total, near_tie_frames=near, bad_frames=bad, worst_margin=worst,
                exact_rate=exact / total, first_stage=first)


def assert_codes_parity(codes_test, codes_ref, margins_ref, margin_tol, min_exact_rate=0.97, what="", **extra):
    r = classify_codes(codes_test, codes_ref, margins_ref, margin_tol)
    # The bar (at most ONE near-tie flip in any comparison, 3999 / 4000
    # frames on config 2, 100 % elsewhere): whatever a caller passes, no more than max(2 frames, 0.5 %) may flip.
    allowed = max(2, int(0.005 * r["total_frames"]))
    min_exact_rate = max(min_exact_rate, 1.0 - allowed / max(1, r["total_frames"]) - 1e-9)
    n_q = int(np.asarray(codes_ref).shape[0])
    first = r["first_stage"]
    # stage-level exact count: every (stage, frame) before a frame's first divergence matches by construction
    stages_exact = int(np.where(first >= 0, first, n_q).sum())
    record_parity(what, kind="codes", frames=r["total_frames"], exact_frames=r["exact_frames"], exact_rate=r["exact_rate"],
                  near_tie_frames=r["near_tie_frames"], bad_frames=r["bad_frames"], worst_accepted_margin=r["worst_margin"],
                  margin_tol=margin_tol, min_exact_rate_asserted=min_exact_rate, n_q=n_q,
                  code_stage_exact_rate=stages_exact / max(1, n_q * r["total_frames"]), **extra)
    assert r["bad_frames"] == 0, f"{what}: {r['bad_frames']} frames differ with oracle margin > {margin_tol} " \
                                  f"(worst {r['worst_margin']:.3e}); exact {r['exact_frames']}/{r['total_frames']}"
    assert r["exact_rate"] >= min_exact_rate, f"{what}: exact-match rate {r['exact_rate']:.4f} < {min_exact_rate}"
    return r
