"""CPU tests of BLASER 2.0: the float64 oracle (oracle/blaser.py) against the golden taken from the reference's own
BlaserModel (tests/golden/blaser_small.pt), the reference unit test's featurization cases, the config, the state-dict
names, the envelope, the ctypes struct layouts, and the kernels' build."""

import ctypes
import os
import re
import shutil
import subprocess
from pathlib import Path

import pytest
import torch

from oracle.blaser import OracleBlaser, featurize, mlp_linear_indices

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = Path(ROOT) / "tests" / "golden" / "blaser_small.pt"


def _golden():
    return torch.load(GOLDEN, weights_only=True)


def test_oracle_matches_the_reference_module():
    g = _golden()
    assert len(g["cases"]) == 3
    for c in g["cases"]:
        o = OracleBlaser(c["state_dict"], input_form=c["input_form"], hidden_dims=c["hidden_dims"], dropout=c["dropout"])
        ref = c["ref"] if c["input_form"] == "COMET" else None
        out = o(c["src"], c["mt"], ref)
        assert out.shape == c["out"].shape == (8, 1)
        torch.testing.assert_close(out, c["out"], rtol=0, atol=1e-6)
        torch.testing.assert_close(o.featurize_input(c["src"], c["mt"], c["ref"]), c["features"], rtol=0, atol=1e-6)
        assert float(c["out"].std()) > 0.1  # the synthetic weights spread the scores
        z = g["zero_row"]
        assert bool(torch.isfinite(c["out"][z]).all()) and float(c["src"][z].abs().max()) == 0.0


@pytest.mark.parametrize("input_form", ["COMET", "QE"])
@pytest.mark.parametrize("embedding_dim", [32, 1024])
def test_oracle_featurization_cases_of_the_reference_unit_test(input_form, embedding_dim):
    """test_blaser_inference.py::test_input_form: how the inputs are concatenated."""
    src = torch.arange(0, embedding_dim).unsqueeze(0) / embedding_dim
    mt, ref = torch.cos(src), torch.exp(src)
    features = featurize(src, mt, ref, input_form)
    if input_form == "COMET":
        expected = [ref, mt, src * mt, ref * mt, torch.absolute(mt - src), torch.absolute(mt - ref)]
    else:
        expected = [src, mt, src * mt, torch.absolute(mt - src)]
    torch.testing.assert_close(features, torch.cat(expected, dim=-1))
    assert features.shape[1] == (6 if input_form == "COMET" else 4) * embedding_dim
    if input_form == "COMET":
        with pytest.raises(ValueError, match="a reference embedding must be provided"):
            featurize(src, mt, None, input_form)


def test_blaser_config_values():
    from sonar_b200 import BlaserConfig, blaser_config

    for arch, form in (("basic_ref", "COMET"), ("basic_qe", "QE")):
        c = blaser_config(arch)
        assert (c.input_form, c.norm_emb, c.embedding_dim, c.output_dim, c.hidden_dims, c.dropout, c.activation,
                c.output_act) == (form, True, 1024, 1, [3072, 1536], 0.1, "TANH", False)
    assert blaser_config("basic_qe", dropout=0.0).dropout == 0.0
    assert BlaserConfig() == blaser_config("basic_ref")  # the dataclass defaults are the basic_ref values
    with pytest.raises(ValueError):
        blaser_config("basic")


def test_state_dict_names_follow_the_module_indices():
    """With dropout the Linear layers of [3072, 1536] are mlp.1 / 4 / 7, without it mlp.0 / 2 / 4; the golden records the
    names the reference module itself gave its Linear layers, also with a hidden size of 0 (skipped)."""
    from sonar_b200.blaser import blaser_config, linear_layer_indices

    assert linear_layer_indices(blaser_config("basic_ref")) == [1, 4, 7]
    assert linear_layer_indices(blaser_config("basic_ref", dropout=0.0)) == [0, 2, 4]
    g = _golden()
    assert len(g["names"]) == 4 and any(0 in n["hidden_dims"] for n in g["names"])
    for c in g["cases"] + g["names"]:
        cfg = blaser_config("basic_ref", input_form=c["input_form"], hidden_dims=c["hidden_dims"], dropout=c["dropout"])
        names = [int(n) for n in c["linear_names"]]
        assert linear_layer_indices(cfg) == names == mlp_linear_indices(c["hidden_dims"], c["dropout"])
    for c in g["cases"]:
        names = [int(n) for n in c["linear_names"]]
        assert {f"mlp.{i}.weight" for i in names} | {f"mlp.{i}.bias" for i in names} == set(c["state_dict"])


def test_envelope_refusals():
    from sonar_b200.blaser import _check_supported, blaser_config

    for ok in (dict(), dict(input_form="QE"), dict(hidden_dims=[256]), dict(hidden_dims=[512, 0, 256]),
               dict(embedding_dim=32), dict(input_form="QE", embedding_dim=16), dict(dropout=0.0)):
        _check_supported(blaser_config("basic_ref", **ok))
    bad = dict(activation="RELU", norm_emb=False, output_act=True, output_dim=2, hidden_dims=[3072, 1000],
               embedding_dim=16)  # 6 * 16 = 96 COMET features: not a multiple of 64
    with pytest.raises(NotImplementedError) as e:
        _check_supported(blaser_config("basic_ref", **bad))
    for field in bad:
        assert field in str(e.value)
    for hidden in ([], [0]):
        with pytest.raises(NotImplementedError, match="hidden layer"):
            _check_supported(blaser_config("basic_ref", hidden_dims=hidden))
    with pytest.raises(NotImplementedError, match="embedding_dim"):
        _check_supported(blaser_config("basic_qe", embedding_dim=24))
    with pytest.raises(ValueError, match="Input form"):
        _check_supported(blaser_config("basic_ref", input_form="XX"))


def test_model_refuses_a_cpu_device_and_load_needs_the_checkpoint(monkeypatch, tmp_path):
    from sonar_b200 import B200BlaserModel, blaser_config, load_blaser_model

    with pytest.raises(RuntimeError, match="CUDA"):
        B200BlaserModel(blaser_config("basic_qe"), {}, device="cpu")
    monkeypatch.setenv("SONAR_B200_CHECKPOINT_DIR", str(tmp_path))
    for name in ("blaser_2_0_ref", "blaser_2_0_qe", "blaser_3"):
        with pytest.raises(FileNotFoundError, match="SONAR_B200_CHECKPOINT_DIR"):
            load_blaser_model(name)


def _header_fields(header, name):
    body = re.search(r"typedef struct " + name + r" \{(.*?)\} " + name + ";", header, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return re.findall(r"(\w+)\s*;", body)


@pytest.mark.parametrize("name", ["SbBlaserConfig", "SbBlaserWeights"])
def test_blaser_ctypes_structs_match_the_header(name, tmp_path):
    from sonar_b200 import _lib

    header = open(os.path.join(ROOT, "include", "sonar_b200.h")).read()
    struct = getattr(_lib, name)
    fields = [f for f, _ in struct._fields_]
    assert fields == _header_fields(header, name)
    for macro in ("SB_EPI_BIAS_TANH", "SB_BLASER_COMET", "SB_BLASER_QE"):
        assert int(re.search(r"#define " + macro + r" (\d+)", header).group(1)) == getattr(_lib, macro)
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler to measure the C layout")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sonar_b200.h"\nint main(void) {\n'
                   f'  printf("%zu\\n", sizeof({name}));\n' +
                   "".join(f'  printf("%zu\\n", offsetof({name}, {f}));\n' for f in fields) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(struct)] + [getattr(struct, f).offset for f in fields]


def _ptxas_blocks(log, pattern):
    return re.findall(r"Function properties for (" + pattern + r")\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads", log)


def test_blaser_kernels_build_without_spills(native_lib):
    """The featurize (4 variants) and output kernels spill nothing, and the tanh GEMM instantiations (EpiMode 7) spill no
    more than the SiLU ones (EpiMode 5) of the same CTA group and output type."""
    from sonar_b200 import build

    assert "blaser.cu" in build.SOURCES and native_lib.sb_version() >= 108
    log = (build.LIB_DIR / "build.log").read_text()
    feat = _ptxas_blocks(log, r"\S*blaser_featurize_kernel\S*")
    outk = _ptxas_blocks(log, r"\S*blaser_output_kernel\S*")
    assert len(feat) == 4 and len(outk) == 1
    for _, frame, st, ld in feat + outk:
        assert (frame, st, ld) == ("0", "0", "0")

    def spills(epi):
        blocks = _ptxas_blocks(log, r"_ZN2sb\w*gemm_bf16_wgmma_kernelILi[12]ELi" + str(epi) + r"E\S*")
        return {name.replace(f"ELi{epi}E", "ELiXE"): int(st) + int(ld) for name, _, st, ld in blocks}

    tanh, silu = spills(7), spills(5)
    assert len(tanh) == 4 and set(tanh) == set(silu)
    for k in tanh:
        assert tanh[k] <= silu[k], (k, tanh[k], silu[k])
