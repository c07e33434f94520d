"""Cascade ST without a GPU: the b200st_cascade_source_args layout against the C header, the exported symbol, a spill-free
handoff kernel, the ASR -> MT vocabulary remap table and the `cascade_st` entry's plan and refusals."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import pytest
import yaml

from neurst_b200 import cli
from neurst_b200 import decode as D
from neurst_b200 import lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cascade_args_layout_matches_the_c_header(tmp_path):
    names = [f for f, _ in L.CascadeSourceArgs._fields_]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200st.h"', 'int main(void) {',
             '  printf("sizeof %zu\\n", sizeof(b200st_cascade_source_args));']
    lines += ['  printf("%s %%zu\\n", offsetof(b200st_cascade_source_args, %s));' % (n, n) for n in names]
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["sizeof"]) == C.sizeof(L.CascadeSourceArgs)
    for n in names:
        assert int(got[n]) == getattr(L.CascadeSourceArgs, n).offset, n


def test_symbol_exported_at_abi_version_203():
    header = open(os.path.join(ROOT, "include", "b200st.h")).read()
    assert "b200st_cascade_source" in L.EXPORTS and re.search(r"\bb200st_cascade_source\s*\(", header)
    assert hasattr(L.load(), "b200st_cascade_source")
    assert L.ABI_VERSION == 203


def test_handoff_kernel_does_not_spill():
    from neurst_b200.csrc import build as B
    from tests.test_kernel_resources_cpu import spill_table
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "cascade.cu"), "-o",
                                                 os.path.join(tmp, "cascade.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    table = {k: v for k, v in spill_table(r.stdout + r.stderr).items() if "cascade_source_kernel" in k}
    assert len(table) == 1 and not any(v[0] or v[1] or v[2] for v in table.values()), table


def test_remap_table_by_token_string():
    t = D.cascade_remap(["a", "b@@", "c", "d"], ["c", "a", "x", "a"], 9, 7)
    # a -> 3 (a later duplicate wins), b@@ missing -> UNK, c -> 0, d missing -> UNK; <UNK>, <SEQ_BEG>, <SEQ_END> -> UNK
    assert t.tolist() == [3, 9, 0, 9, 9, 9, 9] and str(t.dtype) == "torch.int32"
    same = ["w%d" % i for i in range(5)]
    assert D.cascade_remap(same, same, 5, 8).tolist() == [0, 1, 2, 3, 4, 5, 5, 5]        # a shared vocabulary: the identity


def _model_dir(root, name, cls, task_class, task_params, model_params=None):
    d = root / name
    d.mkdir()
    (d / cli.MODEL_CONFIGS).write_text(yaml.safe_dump({"model.class": cls, "model.params": model_params or {},
                                                       "task.class": task_class, "task.params": task_params}))
    return str(d)


def _cascade_cfg(tmp_path, **extra):
    (tmp_path / "vocab.en").write_text("".join("w%d\n" % i for i in range(13)))
    (tmp_path / "vocab.de").write_text("".join("v%d\n" % i for i in range(5)))
    asr = _model_dir(tmp_path, "asr", "SpeechTransformer", "SpeechToText",
                     {"batch_size": 1000, "max_src_len": 400, "max_trg_len": 24,
                      "transcript_data_pipeline.params": {"vocab_path": str(tmp_path / "vocab.en")}})
    mt = _model_dir(tmp_path, "mt", "Transformer", "Seq2Seq",
                    {"src_data_pipeline.params": {"vocab_path": str(tmp_path / "vocab.en")},
                     "trg_data_pipeline.params": {"vocab_path": str(tmp_path / "vocab.de")}})
    cfg = {"entry": "cascade_st", "asr_model_dir": asr, "mt_model_dir": mt, "batch_size": 16,
           "dataset.class": "AudioTripleTFRecordDataset",
           "dataset.params": {"data_path": "DATA", "feature_key": "audio", "transcript_key": "transcript",
                              "translation_key": "translation"},
           "asr_search_method.params": {"beam_size": 4}, "mt_search_method": "beam_search",
           "mt_search_method.params": {"beam_size": 4, "maximum_decode_length": 50}, "asr_output_file": "a.txt"}
    cfg.update(extra)
    return cfg


def test_cascade_plan(tmp_path):
    plan = cli.resolve(_cascade_cfg(tmp_path))
    assert plan["entry"] == "cascade_st" and plan["batch_size"] == 16 and plan["translation_key"] == "translation"
    assert plan["metrics"] == {"asr": "wer", "mt": "bleu"} and plan["asr_output_file"] == "a.txt" and plan["mt_output_file"] is None
    asr, mt = plan["asr"], plan["mt"]
    assert asr["model_class"] == "SpeechTransformer" and mt["model_class"] == "Transformer"
    assert asr["search_method"] == mt["search_method"] == "beam_search"
    assert asr["search"]["beam_size"] == 4 and mt["search"]["maximum_decode_length"] == 50
    assert asr["dataset"] == {"data_path": "DATA", "feature_key": "audio", "transcript_key": "transcript"}
    assert asr["trg_meta"]["vocab_size"] == 16 and mt["src_meta"]["tokens"] == asr["trg_meta"]["tokens"]
    assert asr["batch_size"] == mt["batch_size"] == 16


def test_cascade_refusals(tmp_path):
    with pytest.raises(SystemExit, match="mt_model_dir"):
        cli.resolve({k: v for k, v in _cascade_cfg(tmp_path).items() if k != "mt_model_dir"})
    root = tmp_path / "y"
    root.mkdir()
    cfg = _cascade_cfg(root)
    with pytest.raises(SystemExit, match="AudioTripleTFRecordDataset only"):
        cli.resolve(dict(cfg, **{"dataset.class": "AudioTFRecordDataset"}))
    with pytest.raises(SystemExit, match="not a Transformer"):
        cli.resolve(dict(cfg, mt_model_dir=cfg["asr_model_dir"]))
    with pytest.raises(SystemExit, match="top_sampling"):
        cli.resolve(dict(cfg, asr_search_method="top_sampling"))
    with pytest.raises(SystemExit, match="top_k must be 1"):
        cli.resolve(dict(cfg, **{"asr_search_method.params": {"beam_size": 4, "top_k": 2}}))
    with pytest.raises(SystemExit, match="one device"):
        cli.resolve(cfg, world=2)
    (root / "bare").mkdir()
    (root / "bare" / cli.MODEL_CONFIGS).write_text("model.class: Transformer\n")
    with pytest.raises(SystemExit, match="no task.params"):
        cli.resolve(dict(cfg, mt_model_dir=str(root / "bare")))
