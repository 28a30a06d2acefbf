"""TEST INFRASTRUCTURE ONLY.  Goldens of LFQ tokenizers with large codebooks, from the UNMODIFIED reference
(oracle/ref_loader.py), through the same recipes as oracle/make_golden.py (codes, pre-sign values, taps, reconstruction)
and oracle/make_train_golden.py (eval / train losses and every parameter gradient):

* mini_lfq18 / mini_lfq18_train: ``codebook_size=2**18`` (MAGVIT-v2's vocabulary), 384 latent tokens;
* mini_mc16 / mini_mc16_train: ``codebook_size=2**16, num_codebooks=2, lfq_spherical=True`` (D = 32 projected dims).

The small latent grid (two spatial compressions) keeps the reference's dense (tokens, 2^d) code probabilities to a few GB.

Runs only in the build container:   python -m oracle.make_lfq_large_golden
"""
from __future__ import annotations

from oracle import make_golden as G
from oracle import make_train_golden as TG

LAYERS = ("residual", "compress_space", "compress_space", "compress_time", "residual")

LARGE_CONFIGS = {
    "mini_lfq18": dict(kwargs=dict(image_size=32, init_dim=16, max_dim=64, codebook_size=2 ** 18, layers=LAYERS),
                       video=(2, 3, 5, 32, 32), wseed=0, vseed=1251, full=True),
    "mini_mc16": dict(kwargs=dict(image_size=32, init_dim=16, max_dim=64, codebook_size=2 ** 16, num_codebooks=2, lfq_spherical=True,
                                  layers=LAYERS),
                      video=(2, 3, 5, 32, 32), wseed=0, vseed=1252, full=True),
}


def main():
    G.CONFIGS.update(LARGE_CONFIGS)      # both recipes look their specs up in this table (make_train_golden imports the same dict)
    for name, cfg in LARGE_CONFIGS.items():
        G.make(name)
        TG.make(f"{name}_train", base=name, vseed=cfg["vseed"])


if __name__ == "__main__":
    main()
