"""Generate the committed SigLIP 2 NaFlex fixture (run from the repo root: `python tests/golden/make_golden_naflex.py`).

  tiny_siglip2_naflex/model.safetensors + config.json   a random-init HuggingFace Siglip2Model (16 x 16 position table at patch 4),
                                                        perturbed like the other fixtures (oracle/check_vs_hf.py perturb_)
  tiny_siglip2_naflex/io.npz                            one padded batch in the processor's layout (pixel_values, spatial_shapes,
                                                        pixel_attention_mask; the shapes of naflex_oracle.GOLDEN_SHAPES), token ids,
                                                        and the HuggingFace model's image / text features and logits
The other fixtures are written by make_golden.py and are not touched here.
"""

import os
import sys

os.environ.setdefault("HF_HUB_OFFLINE", "1")
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import check_vs_hf as H  # noqa: E402
import jimm_oracle as O  # noqa: E402
import naflex_oracle as N  # noqa: E402
from make_golden import save  # noqa: E402


def main():
    from transformers import Siglip2Model

    torch.manual_seed(3)
    cfg = N.tiny_siglip2_config()
    m = H.perturb_(Siglip2Model(cfg)).eval()
    with torch.no_grad():
        m.logit_scale.fill_(2.3)
        m.logit_bias.fill_(-1.7)
    oc = N.dual_cfg(cfg)
    P = oc.vision_patch_size
    g = torch.Generator().manual_seed(5)
    images = [torch.rand((h * P, w * P, 3), generator=g) * 2 - 1 for h, w in N.GOLDEN_SHAPES]
    pv, shapes, mask = N.pad_batch(images, P, N.GOLDEN_MAX_PATCHES)
    txt = O.synthetic_tokens(5, oc.context_length, oc.vocab_size, "siglip")
    with torch.no_grad():
        kw = dict(pixel_values=pv, pixel_attention_mask=mask, spatial_shapes=shapes)
        hf_i = m.get_image_features(**kw).pooler_output
        hf_t = m.get_text_features(input_ids=txt).pooler_output
        hf_l = m(input_ids=txt, **kw).logits_per_image
    save("tiny_siglip2_naflex", m, cfg.to_dict(), dict(pixel_values=pv, spatial_shapes=shapes, pixel_attention_mask=mask,
                                                       tokens=txt.to(torch.int32), hf_image_embeds=hf_i, hf_text_embeds=hf_t,
                                                       hf_logits=hf_l))


if __name__ == "__main__":
    main()
