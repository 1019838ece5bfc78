"""Generates tests/golden/extract_reg.npz by running the REFERENCE'S OWN DinoV2ExtractFeatures
(/root/reference/utilities.py, imported verbatim through oracle/reference_import.py) over the DINOv2 backbones with
register tokens, restated in tests/dinov2_reg_restated.py.  Run in the build container only:

    python tests/golden/make_golden_reg.py

The reference passes its model name straight to torch.hub.load (utilities.py:239-240), so "dinov2_vit*14_reg" runs the
class unchanged; its output keeps the 4 register rows after cls (it drops row 0 only, :273).

Per case the file holds the image shape (the image itself is regenerated from seed 1234, see `image`), and per output
(the four facets, and "value_cls_nonorm" = value with use_cls=True, norm_descs=False) a fixed subset of its rows
(`<key>_rows`: the first ones -- cls and registers among them -- then every `step`-th) and of its channels (`cols`).
Every stored element depends on the token order, the positional table and, for the normalised facets, on all channels
of its row; the subsets keep the file small.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import reference_import as ri           # noqa: E402
from tests import dinov2_reg_restated as rr          # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

# tag, model, depth_override, layer, B, H, W, (first rows, row step), channel step.  The 4x5 grid shrinks the 37x37
# positional table, the 38x39 grid enlarges it.
CASES = [
    ("vits14_reg_l9_56x70", "dinov2_vits14_reg", None, 9, 2, 56, 70, (8, 2), 3),
    ("vits14_reg_d2_l1_532x546", "dinov2_vits14_reg", 2, 1, 1, 532, 546, (8, 37), 3),
    ("vitg14_reg_d2_l1_42x42", "dinov2_vitg14_reg", 2, 1, 2, 42, 42, (8, 1), 12),
]
OUTPUTS = [(f, {}) for f in ("value", "key", "query", "token")] + [("value", dict(use_cls=True, norm_descs=False))]


def image(B, H, W):
    return torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(1234))


def rows(n, head, step):
    return np.concatenate([np.arange(min(head, n)), np.arange(head, n, step)]).astype(np.int64)


def main():
    ref = ri.load_reference_utilities()
    out = {}
    for tag, name, depth, layer, B, H, W, (head, step), cstep in CASES:
        model = rr.model(name, depth)
        img = image(B, H, W)
        out[f"{tag}/shape"] = np.array([B, H, W])
        cols = np.arange(0, model.embed_dim, cstep).astype(np.int64)
        out[f"{tag}/cols"] = cols
        for facet, kw in OUTPUTS:
            with ri.hub_patched(lambda n: model):
                ext = ref.DinoV2ExtractFeatures(name, layer, facet, device="cpu", **kw)
            feats = ext(img).numpy()
            key = "value_cls_nonorm" if kw else facet
            r = rows(feats.shape[1], head, step)
            out[f"{tag}/{key}_rows"] = r
            out[f"{tag}/{key}"] = np.ascontiguousarray(feats[:, r][:, :, cols])
    np.savez_compressed(os.path.join(OUT, "extract_reg.npz"), **out)
    print("extract_reg.npz")


if __name__ == "__main__":
    main()
