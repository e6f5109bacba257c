#!/usr/bin/env python
"""Parity report: what the CUDA kernels ACHIEVE, per golden case and per kernel, written as JSON to the path given as the
first argument (default: parity_report.json in the current directory).

    python scripts/parity_report.py [OUT.json]

For every case of tests/golden/golden_v1.npz (outputs of the real reference) and every kernel that supports its plan:
  max |ours - ref32|, the same relative to max(|ref32|, 1), and — in the tolerance units of tests/helpers.py
  (tol = 2e-4 + 1e-4 |truth64| for log-mel / MFCC; the linear-domain amplitude tolerance for spectra) — the worst and the
  99th-percentile distance to the float64 truth of OURS and of the fp32 REFERENCE ITSELF, plus the gate's verdict.
Then BASELINE configs[1] / [2] inputs (8 x 10 s of 0.1 N(0,1)): Fbank-80 and Mfcc(13, 23) against the oracle (bit-pinned to
the reference), with plain allclose-style figures (max abs / max rel) so that the MFCC tolerance of the test-suite is a
measured statement.  Needs an H100; the oracle is the checker (this script is test infrastructure, like tests/)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from helpers import gate_stats, load_golden, oracle_cfg  # noqa: E402
from lhotse_b200 import (B200Fbank, B200FbankConfig, B200LogSpectrogram, B200LogSpectrogramConfig, B200Mfcc,  # noqa: E402
                         B200MfccConfig, B200Spectrogram, B200SpectrogramConfig)
from lhotse_b200.engine import B200FeatError  # noqa: E402
from oracle import kaldi_oracle as O  # noqa: E402

TYPES = {"fbank": (B200Fbank, B200FbankConfig), "mfcc": (B200Mfcc, B200MfccConfig),
         "spectrogram": (B200Spectrogram, B200SpectrogramConfig), "log-spectrogram": (B200LogSpectrogram, B200LogSpectrogramConfig)}


def main():
    rows = []
    for i, c, x, y in load_golden():
        cls, ccls = TYPES[c["feature"]]
        truth = O.extract(x, oracle_cfg(c["feature"], c["cfg"]), dtype=torch.float64)
        sr = c["cfg"].get("sampling_rate", 16000)
        for k in ("generic", "fast", "tc"):
            try:
                ext = cls(ccls(kernel=k, **c["cfg"]))
                ext.engine
            except B200FeatError as e:
                if e.code == -2:
                    continue
                raise
            got = ext.extract(x, sr)
            st = gate_stats(got, y, truth, c["feature"], c["cfg"].get("use_energy", False), c["cfg"].get("use_fft_mag", False))
            st.pop("msg", None)
            rows.append({"case": i, "feature": c["feature"], "kind": c["kind"], "n": c["n"], "N": ext.plan.N, "kernel": k, **st})
    # BASELINE configs[1] / [2] inputs
    torch.manual_seed(1)
    x = (0.1 * torch.randn(8, 160000)).numpy()
    extra = []
    for feature, cls, ccls, cfg, ocfg in (
            ("fbank", B200Fbank, B200FbankConfig, {}, O.OracleConfig()),
            ("mfcc", B200Mfcc, B200MfccConfig, dict(num_ceps=13, num_mel_bins=23), O.OracleConfig(feature="mfcc", num_ceps=13, num_filters=23))):
        for k in ("generic", "fast", "tc"):
            try:
                ext = cls(ccls(kernel=k, **cfg))
                ext.engine
            except B200FeatError as e:
                if e.code == -2:
                    continue
                raise
            got = ext.extract_batch(x, 16000)
            ma, mr, mref, units, runits = 0.0, 0.0, 0.0, 0.0, 0.0
            for b in range(8):
                ref = O.extract(x[b], ocfg)
                truth = O.extract(x[b], ocfg, dtype=torch.float64).astype(np.float64) if hasattr(O.extract(x[b], ocfg, dtype=torch.float64), "astype") else None
                d = np.abs(got[b].astype(np.float64) - ref)
                ma = max(ma, float(d.max()))
                mr = max(mr, float((d / np.maximum(np.abs(ref), 1e-3)).max()))
                # allclose-style: smallest atol that passes at rtol = 1e-3
                mref = max(mref, float((d - 1e-3 * np.abs(ref)).max()))
                st = gate_stats(got[b], ref, truth, feature)
                units, runits = max(units, st["ours_max_units"]), max(runits, st["ref32_max_units"])
                ref_err = float(np.abs(ref.astype(np.float64) - truth).max())
            extra.append({"workload": f"8 x 10 s 0.1*N(0,1), {feature} {cfg}", "kernel": k, "max_abs_diff_vs_ref32": ma,
                          "max_rel_diff_vs_ref32_floor1e-3": mr, "min_atol_at_rtol_1e-3": max(mref, 0.0),
                          "ours_max_units_vs_truth64": units, "ref32_max_units_vs_truth64": runits,
                          "ref32_max_abs_err_vs_truth64_last_cut": ref_err})
    bad = [r for r in rows if not r["ok"]]
    rep = {"gate": {"RTOL": 1e-4, "ATOL": 2e-4, "NOISE_X": 2.0, "neighbourhood": "frame +- 1"},
           "golden_cases": rows, "baseline_inputs": extra,
           "summary": {"cases_x_kernels": len(rows), "failing": len(bad),
                       "worst_ratio_to_limit": max(r["worst_ratio_to_limit"] for r in rows),
                       "worst_ours_units": max(r["ours_max_units"] for r in rows),
                       "worst_ref32_units": max(r["ref32_max_units"] for r in rows),
                       "max_abs_diff_vs_ref32_logmel_mfcc": max(r["max_abs_diff_vs_ref32"] for r in rows if r["feature"] in ("fbank", "mfcc"))}}
    with open(sys.argv[1] if len(sys.argv) > 1 else "parity_report.json", "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep["summary"]))
    for r in bad:
        print("FAIL", r)
    for e in extra:
        print(json.dumps(e))


if __name__ == "__main__":
    main()
