"""Generate the wide sub-band input golden vectors (64 < Isb <= 128) from the UNMODIFIED reference, next to the others.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_wide.py

Same recipe as make_golden.py (whose helpers it uses): the reference model, loaded strictly with the deterministic parameters of
oracle.fsn_oracle.make_params_*, run in float64 one sample per call.  Isb = (2 sb + 1) + k (2 fb + 1), k = 3 for FullSubNet+, 1 for
fullsubnet.Model.  The small configs run on plus_small's inputs (B = 3, F = 33, T = 20) with a sub-band hidden size of 64, so that
the layer-wise tensor-core path takes them.  Writes only
  plus_small_wide70.npz       FullSubNet+, sb 3 / fb 10: Isb 70
  plus_small_wide128.npz      FullSubNet+, sb 2 / fb 20: Isb 128
  plus_small_wide70_GRU.npz   the same as wide70 with sequence_model = "GRU"
  fsn_small_wide66.npz        fullsubnet.Model, cumulative_laplace_norm, sb 20 / fb 12: Isb 66
  fsn_small_wide128.npz       fullsubnet.Model, cumulative_laplace_norm, sb 31 / fb 32: Isb 128
  plus_default_wide124.npz    one 3 s clip at the default geometry (F = 257) with sb 15 / fb 15: Isb 124
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

import make_golden as G  # noqa: E402  (imports the reference, sets up the paths)
from make_golden import O  # noqa: E402

# name: (model kind, config changes, parameter seed, lstm_scale)
SMALL = {
    "plus_small_wide70": ("plus", dict(sb_num_neighbors=3, fb_num_neighbors=10), 21, 1.0),
    "plus_small_wide128": ("plus", dict(sb_num_neighbors=2, fb_num_neighbors=20), 22, 1.0),
    "plus_small_wide70_GRU": ("plus", dict(sb_num_neighbors=3, fb_num_neighbors=10, sequence_model="GRU"), 23, 2.0),
    "fsn_small_wide66": ("fsn", dict(sb_num_neighbors=20, fb_num_neighbors=12), 24, 1.0),
    "fsn_small_wide128": ("fsn", dict(sb_num_neighbors=31, fb_num_neighbors=32), 25, 1.0),
}


def small_cfg(kind, extra):
    c = G.small_plus_cfg() if kind == "plus" else G.small_fsn_cfg("cumulative_laplace_norm")
    c.update(sb_model_hidden_size=64, **extra)
    return c


def main():
    m, r, i = G.small_inputs(3, 33, 20, 7)
    for name, (kind, extra, seed, scale) in SMALL.items():
        cfg = small_cfg(kind, extra)
        if kind == "plus":
            params = O.make_params_plus(cfg, seed=seed, lstm_scale=scale)
            out, _, _ = G.run_plus(cfg, params, m, r, i)
            oo = O.fullsubnet_plus_forward(params, cfg, m, r, i)
        else:
            params = O.make_params_fsn(cfg, seed=seed, lstm_scale=scale)
            out, _ = G.run_fsn(cfg, params, m)
            oo = O.fullsubnet_forward(params, cfg, m)
        print(f"{name}: oracle-vs-reference rel-L2 out={O.rel_l2(oo, out):.2e}")
        G.save(name, out=out, seed=seed, lstm_scale=scale)
    dcfg = O.default_plus_config()
    dcfg.update(sb_num_neighbors=15, fb_num_neighbors=15)
    mag, real, imag, _ = G.spectra(O.synth_clips(1))
    params = O.make_params_plus(dcfg, seed=26)
    out, _, _ = G.run_plus(dcfg, params, mag, real, imag)
    print(f"plus_default_wide124: oracle-vs-reference rel-L2 out={O.rel_l2(O.fullsubnet_plus_forward(params, dcfg, mag, real, imag), out):.2e}")
    G.save("plus_default_wide124", out=out, seed=26)


if __name__ == "__main__":
    main()
