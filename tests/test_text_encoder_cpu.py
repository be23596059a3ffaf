"""CPU: the text encoder's weight inventory against Hugging Face `BertModel`, the host-side checks of a tokenizer batch,
and the conversion of real tokenizer output (a tiny local vocabulary, no download) to sequence lengths."""
import pytest
import torch

from diffuscene_b200.text_encoder import config_geometry, input_lengths, weight_inventory

transformers = pytest.importorskip("transformers")


def test_weight_inventory_matches_bert_state_dict():
    torch.manual_seed(0)
    model = transformers.BertModel(transformers.BertConfig(vocab_size=28996))
    want = [(k, tuple(v.shape)) for k, v in model.state_dict().items() if not k.startswith("pooler.")]
    g = config_geometry(model.config)
    assert (g["layers"], g["hidden"], g["heads"], g["intermediate"]) == (12, 768, 12, 3072)
    assert weight_inventory(g["layers"], g["hidden"], g["intermediate"], g["vocab"], g["max_positions"],
                            g["type_vocab"]) == want


def test_unsupported_semantics_are_rejected():
    for kw in (dict(hidden_act="relu"), dict(layer_norm_eps=1e-5), dict(position_embedding_type="relative_key")):
        with pytest.raises(ValueError):
            config_geometry(transformers.BertConfig(vocab_size=100, **kw))


def test_host_input_checks():
    ids = torch.tensor([[101, 7, 102, 0], [101, 9, 8, 102]])
    mask = torch.tensor([[1, 1, 1, 0], [1, 1, 1, 1]])
    i32, lengths = input_lengths(ids, mask, torch.zeros_like(ids), vocab=200, max_positions=8)
    assert i32.dtype == torch.int32 and torch.equal(i32, ids.int())
    assert lengths.tolist() == [3, 4]
    assert input_lengths(ids, None, None, vocab=200)[1].tolist() == [4, 4]
    bad = [
        dict(input_ids=ids.clone().index_put_((torch.tensor([0]), torch.tensor([1])), torch.tensor(200))),  # id >= vocab
        dict(input_ids=ids.clone().index_put_((torch.tensor([1]), torch.tensor([0])), torch.tensor(-1))),  # id < 0
        dict(input_ids=ids, attention_mask=torch.tensor([[0, 0, 0, 0], [1, 1, 1, 1]])),                    # empty
        dict(input_ids=ids, attention_mask=torch.tensor([[1, 0, 1, 0], [1, 1, 1, 1]])),                    # not a prefix
        dict(input_ids=ids, attention_mask=torch.tensor([[1, 2, 1, 0], [1, 1, 1, 1]])),                    # not 0 / 1
        dict(input_ids=ids, attention_mask=mask[:, :3]),                                                   # wrong shape
        dict(input_ids=ids, attention_mask=mask, token_type_ids=torch.tensor([[0, 0, 1, 0], [0, 0, 0, 0]])),
        dict(input_ids=torch.zeros(2, 9, dtype=torch.int64)),                                              # > max_positions
        dict(input_ids=ids.float()),
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            input_lengths(kw["input_ids"], kw.get("attention_mask"), kw.get("token_type_ids"), vocab=200,
                          max_positions=8)


def test_tokenizer_output_converts_to_lengths(tmp_path):
    words = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", "a", "bed", "desk", "chair", "with", "two", "next", "to",
             "the", "wardrobe", ","]
    vocab = tmp_path / "vocab.txt"
    vocab.write_text("\n".join(words) + "\n")
    tok = transformers.BertTokenizer(vocab_file=str(vocab))
    texts = ["a bed", "a desk with two chair , next to the wardrobe", "wardrobe"]
    enc = tok(texts, return_tensors="pt", padding=True)
    ids, lengths = input_lengths(enc["input_ids"], enc["attention_mask"], enc["token_type_ids"], vocab=len(words),
                                 max_positions=512)
    assert lengths.tolist() == [4, 12, 3]       # [CLS] + words + [SEP]
    assert ids.shape == (3, 12) and int(ids[0, 4:].abs().sum()) == 0       # right-padded with [PAD] = 0
