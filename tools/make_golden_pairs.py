"""Record the reference's scene graphs and pairwise-inference entry order as tests/golden/pairs.json.

Needs a reference checkout: $SPANN3R_REFERENCE, else a `reference` directory next to this repository.  Only the JSON
it writes is committed; tests/test_offline_cpu.py checks `spann3r_b200.offline.make_pairs` / `inference` against it.

  python tools/make_golden_pairs.py

"graphs": for F in {1, 2, 5, 7} x scene graph x symmetrize x prefilter, the (idx1, idx2) list of
dust3r.image_pairs.make_pairs, or the exception type it raised.
"entries": for F in {4, 5} and batch_size in {2, 3}, the view1 / view2 idx lists that dust3r.inference.inference
returns for make_pairs(complete, symmetrize=True): each batch collated by collate_with_cat and symmetrised by
_interleave_imgs, on dummy tensors (no model runs).
"""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("SPANN3R_REFERENCE") or os.path.join(os.path.dirname(REPO), "reference")

GRAPHS = ["swin", "swin-2", "oneref", "oneref-3", "prev", "complete"]
PREFILTERS = [None, "seq1", "cyc2"]


def views(n):
    return [{"img": torch.full((1, 3, 2, 2), float(i)), "true_shape": torch.tensor([[2, 2]]), "idx": i, "instance": str(i)}
            for i in range(n)]


def main():
    sys.path.insert(0, REF)
    from dust3r.image_pairs import make_pairs                      # noqa (reference)
    from dust3r.inference import make_batch_symmetric              # noqa (reference)
    from dust3r.utils.device import collate_with_cat               # noqa (reference)

    graphs = []
    for n in (1, 2, 5, 7):
        for g in GRAPHS:
            for sym in (True, False):
                for pf in PREFILTERS:
                    case = {"n": n, "scene_graph": g, "symmetrize": sym, "prefilter": pf}
                    try:
                        case["pairs"] = [[a["idx"], b["idx"]] for a, b in make_pairs(views(n), g, pf, sym)]
                    except Exception as ex:  # noqa: BLE001 -- the kind of failure is the recorded result
                        case["raises"] = type(ex).__name__
                    graphs.append(case)

    entries = []
    for n in (4, 5):
        pairs = make_pairs(views(n), "complete", None, True)
        for bs in (2, 3):
            v1, v2 = [], []
            for i in range(0, len(pairs), bs):
                a, b = make_batch_symmetric(collate_with_cat(pairs[i:i + bs]))
                v1 += list(a["idx"])
                v2 += list(b["idx"])
            entries.append({"n": n, "batch_size": bs, "view1_idx": v1, "view2_idx": v2})

    out = os.path.join(REPO, "tests", "golden", "pairs.json")
    with open(out, "w") as f:
        json.dump({"graphs": graphs, "entries": entries}, f, indent=0)
        f.write("\n")
    print("wrote", out, len(graphs), "graph cases,", len(entries), "entry orders")


if __name__ == "__main__":
    main()
