"""Cascade ST on the device: the handoff kernel (b200st_cascade_source) against a host restatement on empty hypotheses,
hypotheses that reach the maximum length, missing tokens and truncation, its refusals before any launch, and the
`cascade_st` entry's MT hypotheses identical to `predict` of the MT model over a processed-text file of the ASR output."""
import pytest
import torch

from neurst_b200 import cli
from neurst_b200 import decode as D
from neurst_b200 import lib as L
from tests import parity_utils as U
from tests.test_cli import _write_dataset, _write_yaml

pytestmark = pytest.mark.gpu


def _restated(hyp, remap, asr_eos, asr_vocab, mt_eos, mt_pad, mt_unk, max_src_len):
    rows = []
    for r in hyp.tolist():
        n = r.index(asr_eos) if asr_eos in r else len(r)
        ids = [remap[i] if 0 <= i < asr_vocab else mt_unk for i in r[:n]] + [mt_eos]
        if max_src_len and len(ids) > max_src_len:
            ids = ids[:max_src_len - 1] + ids[-1:]
        rows.append(ids)
    T = max(len(r) for r in rows)
    return ([r + [mt_pad] * (T - len(r)) for r in rows], [[0.0] * len(r) + [1.0] * (T - len(r)) for r in rows],
            [len(r) for r in rows])


@pytest.mark.parametrize("max_src_len", [0, 5])
def test_handoff_edge_cases(max_src_len):
    asr_vocab, asr_eos = 12, 11
    remap = D.cascade_remap(["a", "b", "c", "d", "e", "f", "g", "h", "i"], ["i", "h", "g", "f", "e", "d", "c", "b"], 7, asr_vocab)
    L_ = 9
    hyp = torch.full((5, L_), asr_eos, dtype=torch.long)
    hyp[1] = torch.tensor([0, 1, 2, 3, 4, 5, 6, 7, 1])                      # reaches the maximum length, no EOS
    hyp[2, :4] = torch.tensor([8, 0, 40, -3])                              # "a" missing from the MT vocabulary; ids out of range
    hyp[3, :3] = torch.tensor([2, 2, 9])                                   # <UNK> of the ASR side
    hyp[4, :6] = torch.tensor([3, 4, 5, 6, 7, 0])                          # truncated when max_src_len = 5
    hyp[4, 7] = 2                                                          # past the first EOS: ignored
    src, pad, length = D.cascade_source(hyp.cuda(), remap, asr_eos, 9, 8, 8, 7, max_src_len=max_src_len)
    torch.cuda.synchronize()
    want_ids, want_pad, want_len = _restated(hyp, remap.tolist(), asr_eos, asr_vocab, 8, 8, 7, max_src_len)
    assert src.cpu().tolist() == want_ids and pad.cpu().tolist() == want_pad and length.cpu().tolist() == want_len
    assert want_len[0] == 1 and want_ids[2][:4] == [0, 7, 7, 7]


def test_handoff_refuses_bad_tables_and_ids_before_launch():
    hyp = torch.zeros(2, 4, dtype=torch.long, device="cuda")
    before = int(L.load().b200st_launch_count())
    with pytest.raises(L.B200STError, match="outside the MT vocabulary"):
        D.cascade_source(hyp, torch.tensor([0, 9], dtype=torch.int32), 1, 9, 8, 8, 7)
    for bad in (dict(asr_eos_id=2), dict(mt_eos_id=9), dict(mt_unk_id=-1)):
        kw = dict(asr_eos_id=1, mt_vocab=9, mt_eos_id=8, mt_pad_id=8, mt_unk_id=7)
        kw.update(bad)
        with pytest.raises(L.B200STError, match="check failed"):
            D.cascade_source(hyp, torch.tensor([0, 1], dtype=torch.int32), **kw)
    assert int(L.load().b200st_launch_count()) == before


TINY = {"encoder.num_layers": 2, "decoder.num_layers": 2, "encoder.hidden_size": 128, "decoder.hidden_size": 128, "modality.dim": 128,
        "encoder.num_attention_heads": 2, "decoder.num_attention_heads": 2, "encoder.filter_size": 256, "decoder.filter_size": 256}


def _save(plan, model, model_dir):
    plan = dict(plan, model_dir=model_dir)
    P = U.chaotic_decode_params({k: v.detach().cpu() for k, v in model.named_parameters().items()}, 4.0, 3)
    model.load_parameters(P)
    cli.write_model_configs(plan)
    cli.save_checkpoint(model.runtime, model_dir, 1)


def test_cascade_mt_hypotheses_equal_predict_over_the_asr_output(tmp_path):
    _write_dataset(tmp_path, n_shards=1, per_shard=40, vocab=93)
    y = _write_yaml(tmp_path, data=str(tmp_path / "train.tfrecords"), n_tokens=93)
    asr_cfg = cli.load_config([y], [("task.params.max_src_len", 400), ("task.params.max_trg_len", 24),
                                    ("model.params.modality.source.channels", 64)] + [("model.params." + k, v) for k, v in TINY.items()])
    asr_plan = cli.resolve(asr_cfg)
    _save(asr_plan, cli._build_model(asr_plan).init_parameters(1), str(tmp_path / "asr"))
    # MT source vocabulary: the ASR tokens tok0..tok79 (tok80..tok92 become UNK) and a few of its own; 88 entries
    (tmp_path / "mt.src").write_text("".join("tok%d\n" % i for i in range(80)) + "".join("x%d\n" % i for i in range(5)))
    (tmp_path / "mt.trg").write_text("".join("y%d\n" % i for i in range(45)))
    mt_cfg = {"task.class": "seq2seq", "hparams_set": "transformer_s", "model.params": TINY,
              "task.params": {"batch_size": 100, "src_data_pipeline.params": {"vocab_path": str(tmp_path / "mt.src")},
                              "trg_data_pipeline.params": {"vocab_path": str(tmp_path / "mt.trg")}},
              "dataset.params": {"src_file": str(tmp_path / "mt.src"), "data_is_processed": True}}
    mt_plan = cli.resolve(mt_cfg)
    _save(mt_plan, cli._build_model(mt_plan).init_parameters(2), str(tmp_path / "mt"))
    search = {"beam_size": 4, "maximum_decode_length": 30}
    cfg = {"entry": "cascade_st", "asr_model_dir": str(tmp_path / "asr"), "mt_model_dir": str(tmp_path / "mt"), "batch_size": 16,
           "dataset.params": {"data_path": str(tmp_path / "train.tfrecords"), "transcript_key": "translation",
                              "translation_key": "translation"},
           "asr_search_method.params": search, "mt_search_method.params": search,
           "asr_output_file": str(tmp_path / "asr.txt"), "mt_output_file": str(tmp_path / "mt.txt")}
    res = cli.cascade_st(cli.resolve(cfg))
    assert len(res["asr_hypotheses"]) == len(res["mt_hypotheses"]) == 40 and "asr_metric" in res
    # predict of the ASR model, then predict of the MT model over the ASR output as processed text
    asr_pred = cli.predict(cli.resolve(dict(asr_cfg, **{"entry.class": "predict", "model_dir": str(tmp_path / "asr"), "batch_size": 16,
                                                        "search_method": "beam_search", "search_method.params": search})))
    asr_text = [t for t, _ in asr_pred["hypotheses"]]
    assert asr_text == res["asr_hypotheses"]
    (tmp_path / "asr_bpe.txt").write_text("".join(t + "\n" for t in asr_text))
    mt_pred = cli.predict(cli.resolve(dict(mt_cfg, **{"entry.class": "predict", "model_dir": str(tmp_path / "mt"), "batch_size": 16,
                                                      "search_method": "beam_search", "search_method.params": search,
                                                      "dataset.params": {"src_file": str(tmp_path / "asr_bpe.txt"),
                                                                         "data_is_processed": True}})))
    assert [t for t, _ in mt_pred["hypotheses"]] == res["mt_hypotheses"]
    assert open(tmp_path / "mt.txt").read().splitlines() == res["mt_hypotheses"]
    assert len(set(res["mt_hypotheses"])) > 1
