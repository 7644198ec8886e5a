"""Generate tests/golden/blaser_small.pt from the reference's OWN BlaserModel (sonar/models/blaser/model.py), loaded by
file path -- the module imports only torch -- and built with its own constructor, so the golden pins both the arithmetic
of oracle/blaser.py and the reference's `mlp.<i>` parameter names (Dropout modules shift them when dropout > 0).

    python tests/golden/make_blaser_golden.py <SONAR checkout>/sonar/models/blaser/model.py

Weights and inputs follow the recipe of oracle/blaser.py (scores spread, not the near-constant default init).  The
weights are rounded to bf16 values and stored as bf16, which halves the file; the module runs in float64 on exactly those
values.  Row 3 of every input is all zeros (F.normalize keeps it zero).  The parameter names need no weights: `names`
records the Linear layers of modules built with the card's hidden sizes and with a hidden size of 0, which the reference
skips."""

import importlib.util
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle.blaser import make_blaser_inputs, make_synthetic_blaser_state_dict  # noqa: E402

# (input_form, embedding_dim, hidden_dims, dropout): hidden sizes of 256, the smallest the engine runs
CASES = [("COMET", 32, [256, 256], 0.1), ("QE", 32, [256], 0.0), ("QE", 64, [256], 0.1)]
# (input_form, hidden_dims, dropout) of the modules whose Linear names are recorded
NAME_CASES = [("COMET", [3072, 1536], 0.1), ("QE", [3072, 1536], 0.0), ("COMET", [256, 0, 256], 0.1),
              ("QE", [256, 0, 256], 0.0)]
ROWS = 8
ZERO_ROW = 3


def _build(mod, form, e, hidden, dropout):
    return mod.BlaserModel(embedding_dim=e, output_dim=1, hidden_dims=hidden, dropout=dropout, activation="TANH",
                           input_form=form, norm_emb=True, output_act=False).eval()


def _linear_names(model):
    return [n for n, m in model.mlp.named_children() if isinstance(m, torch.nn.Linear)]


def main() -> None:
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    spec = importlib.util.spec_from_file_location("blaser_model", sys.argv[1])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    cases = []
    for i, (form, e, hidden, dropout) in enumerate(CASES):
        model = _build(mod, form, e, hidden, dropout)
        sd = {k: v.to(torch.bfloat16) for k, v in make_synthetic_blaser_state_dict(form, e, hidden, dropout,
                                                                                   seed=100 + i).items()}
        model.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)  # only the module's own names load
        src, mt, ref = make_blaser_inputs(ROWS, e, seed=200 + i)
        for t in (src, mt, ref):
            t[ZERO_ROW] = 0.0
        model = model.double()
        with torch.no_grad():
            d = (src.double(), mt.double(), ref.double())
            out = model(src=d[0], mt=d[1], ref=d[2])
            feats = model.featurize_input(src=d[0], mt=d[1], ref=d[2])
        cases.append({"input_form": form, "embedding_dim": e, "hidden_dims": hidden, "dropout": dropout,
                      "linear_names": _linear_names(model), "state_dict": sd, "src": src, "mt": mt, "ref": ref,
                      "features": feats, "out": out})
    names = [{"input_form": form, "hidden_dims": hidden, "dropout": dropout,
              "linear_names": _linear_names(_build(mod, form, 32, hidden, dropout))} for form, hidden, dropout in NAME_CASES]
    torch.save({"cases": cases, "names": names, "zero_row": ZERO_ROW,
                "generator": "sonar/models/blaser/model.py BlaserModel (float64)"}, os.path.join(HERE, "blaser_small.pt"))
    print("wrote blaser_small.pt", [tuple(c["out"].shape) for c in cases], [n["linear_names"] for n in names])


if __name__ == "__main__":
    main()
