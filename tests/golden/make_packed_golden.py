"""Generate tests/golden/ref_packed_docs.pt from the reference's OWN code (run where /root/reference is mounted):
    python tests/golden/make_packed_golden.py

The fixture holds, for seeded EOD-delimited token rows (tests/test_packed_docs_host.py::golden_token_rows), what the
reference's get_ltor_masks_and_position_ids(reset_position_ids=True, reset_attention_mask=True)
(long_vita_megatron/training/utils.py:192-249) returns - the [S, S] attention mask and the position ids - and what its
compute_actual_seq_len (:53-57) makes of those position ids.  Machines without the reference read the file only.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import test_packed_docs_host as TD  # noqa: E402


def main():
    out = os.path.join(HERE, "ref_packed_docs.pt")
    torch.save(TD.reference_packed_docs(), out)
    print("wrote", out)


if __name__ == "__main__":
    main()
