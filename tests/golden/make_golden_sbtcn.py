"""Generate the sub-band TCN golden vectors (sequence_model = "TCN") from the UNMODIFIED reference, next to the others.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_sbtcn.py

Same recipe as make_golden.py (whose helpers it uses): the reference's FullSubNet_Plus, loaded strictly with the deterministic
parameters of tests/sbtcn_oracle.make_params, run in float64 one sample per call.  Writes only
  plus_small_sbTCN.npz    small config (F = 33, Isb = 10) on plus_small's inputs: out, fb_out, sb_in
  plus_default_sbTCN.npz  one 3 s clip at the default geometry (F = 257, Isb = 34): out
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

import make_golden as G  # noqa: E402  (imports the reference, sets up the paths)
import sbtcn_oracle as S  # noqa: E402
from make_golden import O  # noqa: E402


def main():
    tcfg = dict(G.small_plus_cfg(), sequence_model="TCN")
    m, r, i = G.small_inputs(3, 33, 20, 7)
    params = S.make_params(tcfg, seed=15)
    out, fb_in, fb_out = G.run_plus(tcfg, params, m, r, i)
    st = {}
    oo = S.forward(params, tcfg, m, r, i, stages=st)
    print(f"plus_small[sub-band TCN]: oracle-vs-reference rel-L2 out={O.rel_l2(oo, out):.2e} fb_out={O.rel_l2(st['fb_out'], fb_out):.2e}")
    G.save("plus_small_sbTCN", out=out, fb_out=fb_out, sb_in=st["sb_in"], seed=15)
    dcfg = dict(O.default_plus_config(), sequence_model="TCN")
    mag, real, imag, _ = G.spectra(O.synth_clips(1))
    params = S.make_params(dcfg, seed=0)
    out, _, _ = G.run_plus(dcfg, params, mag, real, imag)
    print(f"plus_default[sub-band TCN]: oracle-vs-reference rel-L2 out={O.rel_l2(S.forward(params, dcfg, mag, real, imag), out):.2e}")
    G.save("plus_default_sbTCN", out=out, seed=0)


if __name__ == "__main__":
    main()
