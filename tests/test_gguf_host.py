"""GGUF reader, dequantization restatement, tokenizer rebuild and embedder-string resolver on the host (no GPU)."""

from __future__ import annotations

import struct

import numpy as np
import pytest
from gguf_fixtures import (
    ARR, BOOL, F16, F32, F32V, F64, I8, I16, I32, I64, Q4_K, Q6_K, Q8_0, STR, U8, U16, U32, U64, dequant, random_blocks,
    unigram_metadata, write_gguf,
)

from raglite_b200._gguf import GGUFFile, bert_plan, find_cached_gguf, gguf_tokenizer, parse_embedder

META = [("u8", U8, 7), ("i8", I8, -7), ("u16", U16, 65535), ("i16", I16, -32768), ("u32", U32, 2**32 - 1),
        ("i32", I32, -(2**31)), ("f32", F32V, 1.5), ("b", BOOL, True), ("s", STR, "héllo ⊕"), ("u64", U64, 2**64 - 1),
        ("i64", I64, -(2**63)), ("f64", F64, 0.1), ("astr", ARR, (STR, ["a", "", "▁b"])), ("ai32", ARR, (I32, [1, -2, 3])),
        ("af32", ARR, (F32V, [0.5, -1.0])), ("anest", ARR, (ARR, [(U8, [1, 2]), (U8, [])]))]


@pytest.mark.parametrize("alignment", [32, 64])
@pytest.mark.parametrize("version", [2, 3])
def test_reader_round_trip(tmp_path, alignment, version) -> None:  # noqa: ANN001
    rng = np.random.default_rng(0)
    tensors = [("w_f32", F32, (3, 5), random_blocks(F32, 3, 5, rng)), ("w_f16", F16, (2, 8), random_blocks(F16, 2, 8, rng)),
               ("q8", Q8_0, (2, 64), random_blocks(Q8_0, 2, 64, rng)), ("q4", Q4_K, (3, 256), random_blocks(Q4_K, 3, 256, rng)),
               ("q6", Q6_K, (1, 512), random_blocks(Q6_K, 1, 512, rng)), ("bias", F32, (7,), random_blocks(F32, 1, 7, rng))]
    path = tmp_path / "t.gguf"
    write_gguf(path, META, [(n, t, s, r.tobytes()) for n, t, s, r in tensors], alignment=alignment, version=version)
    f = GGUFFile(path)
    assert f.version == version and f.alignment == alignment
    for k, _, v in META:
        got = f.metadata[k]
        if isinstance(v, tuple):
            want = v[1] if v[0] != ARR else [w[1] for w in v[1]]
            got = [list(g) for g in got] if v[0] == ARR else list(got)
            assert got == pytest.approx(want) if v[0] == F32V else got == want
        elif isinstance(v, float):
            assert got == pytest.approx(v)
        else:
            assert got == v
    for n, t, s, r in tensors:
        assert f.tensors[n].ggml_type == t and f.tensors[n].shape == s
        assert np.array_equal(f.tensors[n].data, r)
    body = path.read_bytes()
    for _, _, _, r in tensors:   # each tensor's bytes start on an alignment boundary of the file
        assert body.find(r.tobytes()) % alignment == 0


def test_reader_matches_gguf_writer(tmp_path) -> None:  # noqa: ANN001
    gguf = pytest.importorskip("gguf")
    rng = np.random.default_rng(1)
    path = tmp_path / "w.gguf"
    w = gguf.GGUFWriter(str(path), "bert")
    w.add_block_count(2)
    w.add_string("x.s", "abc")
    w.add_array("x.a", ["p", "q"])
    w.add_precompiled_charsmap(b"\x01\x02\x03")
    raw = {"q4": (Q4_K, random_blocks(Q4_K, 4, 256, rng)), "q8": (Q8_0, random_blocks(Q8_0, 2, 64, rng)),
           "f": (F32, random_blocks(F32, 3, 4, rng))}
    shapes = {"q4": (4, 256), "q8": (2, 64), "f": (3, 4)}
    for n, (t, r) in raw.items():
        w.add_tensor(n, r.reshape(shapes[n][0], -1), raw_dtype=gguf.GGMLQuantizationType(t))
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    f = GGUFFile(path)
    ref = gguf.GGUFReader(str(path))
    assert f.get("general.architecture") == "bert" and f.get("bert.block_count") == 2 and f.get("x.s") == "abc"
    assert list(f.get("x.a")) == ["p", "q"] and bytes(f.get("tokenizer.ggml.precompiled_charsmap")) == b"\x01\x02\x03"
    for t in ref.tensors:
        assert f.tensors[t.name].shape == shapes[t.name]
        assert np.array_equal(f.tensors[t.name].data, np.asarray(t.data).reshape(-1).view(np.uint8))


def test_malformed_files_raise(tmp_path) -> None:  # noqa: ANN001
    rng = np.random.default_rng(2)
    path = tmp_path / "m.gguf"
    write_gguf(path, META[:3], [("q", Q4_K, (2, 256), random_blocks(Q4_K, 2, 256, rng).tobytes())])
    good = path.read_bytes()
    cases = {"bad magic": b"GGUG" + good[4:], "version": good[:4] + struct.pack("<I", 4) + good[8:],
             "truncated header": good[:40], "past the end": good[:-10], "empty": b""}
    for what, data in cases.items():
        path.write_bytes(data)
        with pytest.raises(ValueError):
            GGUFFile(path)
    write_gguf(path, [], [("bf", 30, (2, 32), b"\0" * 128)])
    with pytest.raises(ValueError, match="'bf'.*30"):
        GGUFFile(path)


def _q4k_block(d: float, dmin: float, scales: list[int], mins: list[int], nibbles: np.ndarray) -> np.ndarray:
    """One Q4_K block from its 8 scales / mins (6 bits each) in ggml's 12-byte packing and 256 nibbles (ggml order)."""
    s = np.zeros(12, np.uint8)
    for j in range(8):
        if j < 4:
            s[j] |= scales[j]
            s[j + 4] |= mins[j]
        else:
            s[j + 4] = (scales[j] & 0xF) | ((mins[j] & 0xF) << 4)
            s[j - 4] |= (scales[j] >> 4) << 6
            s[j] |= (mins[j] >> 4) << 6
    qs = np.zeros(128, np.uint8)
    for j64 in range(4):
        qs[32 * j64:32 * j64 + 32] = nibbles[64 * j64:64 * j64 + 32] | (nibbles[64 * j64 + 32:64 * j64 + 64] << 4)
    return np.concatenate([np.array([d, dmin], np.float16).view(np.uint8), s, qs])


def test_dequant_hand_built_blocks() -> None:
    nib = np.tile(np.array([0, 15, 1, 14], np.uint8), 64)
    sc, mn = [1, 2, 3, 63, 17, 33, 48, 63], [0, 63, 5, 9, 31, 32, 62, 1]
    y = dequant(Q4_K, _q4k_block(0.5, 0.25, sc, mn, nib), 1, 256)[0]
    for j in range(8):   # both halves of the 6-bit packing, nibbles 0 and 15
        j64, hi = divmod(j, 2)
        e = 64 * j64 + 32 * hi
        want = np.float32(0.5) * np.float32(sc[j]) * nib[e:e + 32].astype(np.float32) - np.float32(0.25) * np.float32(mn[j])
        assert np.array_equal(y[e:e + 32], want)
    # Q6_K: negative scales, q = 0 and 63
    b = np.zeros(210, np.uint8)
    b[:128] = 0xF0
    b[128:192] = 0b11001100
    b[192:208] = np.array([-128, -1, 1, 127] * 4, np.int8).view(np.uint8)
    b[208:210] = np.array([2.0 ** -24], np.float16).view(np.uint8)   # subnormal fp16 d
    y = dequant(Q6_K, b, 1, 256)[0]
    d = np.float32(2.0 ** -24)
    # element 0: q = 0, sc[0] = -128; 32: q = 48, sc[2] = 1; 64: q = 15, sc[4] = -128; 96: q = 63, sc[6] = 1
    assert [y[0], y[32], y[64], y[96]] == [(d * -128) * -32, d * 16, (d * -128) * -17, d * 31]
    q8 = np.concatenate([np.array([-3.0], np.float16).view(np.uint8), np.arange(-16, 16, dtype=np.int8).view(np.uint8)])
    assert np.array_equal(dequant(Q8_0, q8, 1, 32)[0], np.float32(-3.0) * np.arange(-16, 16, dtype=np.float32))


@pytest.mark.parametrize("ty", [Q8_0, Q4_K, Q6_K])
def test_dequant_matches_gguf_package(ty) -> None:  # noqa: ANN001
    gguf = pytest.importorskip("gguf")
    from gguf.quants import dequantize

    rng = np.random.default_rng(ty)
    raw = random_blocks(ty, 64, 1024, rng, scale=50.0)
    want = dequantize(raw.reshape(64, -1), gguf.GGMLQuantizationType(ty)).astype(np.float32)
    assert np.array_equal(dequant(ty, raw, 64, 1024).view(np.uint32), want.view(np.uint32))


TEXTS = ["", "a⊕b ⊕ c", "two  spaces   three    four", "tab\there\nnew line\r\n", "café naïve Ünïcödé",
         "中文字符 日本語 한국어", "  leading and trailing  ", "ＦＵＬＬ ｗｉｄｔｈ ①②", "The observer's clock."]


def _roundtrip(tmp_path, tok, **kw):  # noqa: ANN001, ANN003, ANN202
    path = tmp_path / "tok.gguf"
    write_gguf(path, [("general.architecture", STR, "bert"), *unigram_metadata(tok, **kw)], [])
    return gguf_tokenizer(GGUFFile(path))


def test_tokenizer_rebuild_unigram(tmp_path) -> None:  # noqa: ANN001
    from oracle.embed import unigram_tokenizer

    tok = unigram_tokenizer()
    rebuilt = _roundtrip(tmp_path, tok, remove_extra_ws=False)
    for s in TEXTS:
        assert rebuilt.encode(s).ids == tok.encode(s).ids, s


def test_tokenizer_rebuild_sentencepiece_nmt_nfkc(tmp_path) -> None:  # noqa: ANN001
    """A SentencePiece Unigram model trained here with nmt_nfkc (a real precompiled charsmap), written as GGUF metadata:
    the rebuilt tokenizer gives SentencePiece's own ids.  Trailing whitespace is left out: SentencePiece strips it,
    while the Precompiled + Replace pipeline of bge-m3's tokenizer.json keeps one trailing piece."""
    spm = pytest.importorskip("sentencepiece")
    from sentencepiece import sentencepiece_model_pb2 as pb

    corpus = tmp_path / "c.txt"
    rng = np.random.default_rng(0)
    words = ["light", "clock", "observer", "café", "naïve", "中文", "字符", "time", "frame", "⊕", "event", "ＦＵＬＬ"]
    corpus.write_text("\n".join(" ".join(rng.choice(words, 8)) for _ in range(2000)))
    prefix = str(tmp_path / "sp")
    spm.SentencePieceTrainer.train(input=str(corpus), model_prefix=prefix, vocab_size=50, model_type="unigram",
                                   hard_vocab_limit=False, normalization_rule_name="nmt_nfkc", character_coverage=1.0)
    sp = spm.SentencePieceProcessor(model_file=prefix + ".model")
    m = pb.ModelProto()
    m.ParseFromString(open(prefix + ".model", "rb").read())  # noqa: SIM115
    assert len(m.normalizer_spec.precompiled_charsmap) > 0
    md = [("tokenizer.ggml.model", STR, "t5"), ("tokenizer.ggml.tokens", ARR, (STR, [p.piece for p in m.pieces])),
          ("tokenizer.ggml.scores", ARR, (F32V, [p.score for p in m.pieces])),
          ("tokenizer.ggml.unknown_token_id", U32, sp.unk_id()), ("tokenizer.ggml.bos_token_id", U32, sp.bos_id()),
          ("tokenizer.ggml.eos_token_id", U32, sp.eos_id()), ("tokenizer.ggml.add_space_prefix", BOOL, True),
          ("tokenizer.ggml.remove_extra_whitespaces", BOOL, True),
          ("tokenizer.ggml.precompiled_charsmap", ARR, (U8, list(m.normalizer_spec.precompiled_charsmap)))]
    path = tmp_path / "t.gguf"
    write_gguf(path, md, [])
    rebuilt = gguf_tokenizer(GGUFFile(path))
    for s in TEXTS:
        s = s.rstrip()
        assert rebuilt.encode(s).ids == [sp.bos_id(), *sp.encode(s), sp.eos_id()], s


def test_tokenizer_other_models_raise(tmp_path) -> None:  # noqa: ANN001
    path = tmp_path / "b.gguf"
    write_gguf(path, [("tokenizer.ggml.model", STR, "bert")], [])
    with pytest.raises(ValueError, match="tokenizer.json"):
        gguf_tokenizer(GGUFFile(path))


def test_resolver(tmp_path) -> None:  # noqa: ANN001
    e = "llama-cpp-python/lm-kit/bge-m3-gguf/*F16.gguf@512"
    assert parse_embedder(e) == ("lm-kit/bge-m3-gguf", "*F16.gguf", 512)
    assert parse_embedder("llama-cpp-python/lm-kit/bge-m3-gguf/*Q4_K_M.gguf") == ("lm-kit/bge-m3-gguf", "*Q4_K_M.gguf", 0)
    root = tmp_path / "models--lm-kit--bge-m3-gguf" / "snapshots"
    with pytest.raises(FileNotFoundError, match="no file"):
        find_cached_gguf("lm-kit/bge-m3-gguf", "*F16.gguf", tmp_path)
    (root / "s1").mkdir(parents=True)
    (root / "s1" / "bge-m3-F16.gguf").write_bytes(b"x")
    (root / "s1" / "bge-m3-Q4_K_M.gguf").write_bytes(b"y")
    assert find_cached_gguf("lm-kit/bge-m3-gguf", "*F16.gguf", tmp_path) == root / "s1" / "bge-m3-F16.gguf"
    (root / "s2").mkdir()
    (root / "s2" / "other-F16.gguf").write_bytes(b"z")
    with pytest.raises(FileNotFoundError, match="2 files.*bge-m3-Q4_K_M"):
        find_cached_gguf("lm-kit/bge-m3-gguf", "*F16.gguf", tmp_path)


def _bert_file(tmp_path, **over):  # noqa: ANN001, ANN003, ANN202
    md = {"general.architecture": (STR, "bert"), "bert.block_count": (U32, 1), "bert.embedding_length": (U32, 64),
          "bert.feed_forward_length": (U32, 128), "bert.attention.head_count": (U32, 1),
          "bert.attention.layer_norm_epsilon": (F32V, 1e-5), "bert.context_length": (U32, 512)}
    md.update(over)
    path = tmp_path / "b.gguf"
    write_gguf(path, [(k, t, v) for k, (t, v) in md.items()], [("token_embd.weight", F16, (10, 64), b"\0" * 1280)])
    return GGUFFile(path)


def test_plan_errors_before_any_device_work(tmp_path) -> None:  # noqa: ANN001
    with pytest.raises(ValueError, match="nomic-bert"):
        bert_plan(_bert_file(tmp_path, **{"general.architecture": (STR, "nomic-bert")}))
    with pytest.raises(ValueError, match="head_dim"):
        bert_plan(_bert_file(tmp_path, **{"bert.attention.head_count": (U32, 4)}))
    with pytest.raises(ValueError, match="hidden"):
        bert_plan(_bert_file(tmp_path, **{"bert.embedding_length": (U32, 2048), "bert.attention.head_count": (U32, 32)}))
    with pytest.raises(ValueError, match="position_embd"):
        bert_plan(_bert_file(tmp_path))
    with pytest.raises(ValueError, match="3 tokens but token_embd has 10"):
        bert_plan(_bert_file(tmp_path, **{"tokenizer.ggml.tokens": (ARR, (STR, ["a", "b", "c"]))}))


def _tiny_bert(tmp_path, H: int, F: int, linear_type: int):  # noqa: ANN001, ANN202
    """A complete one-layer ``bert`` file whose four projections have ``linear_type`` (the rest F32)."""
    rng = np.random.default_rng(3)
    md = [("general.architecture", STR, "bert"), ("bert.block_count", U32, 1), ("bert.embedding_length", U32, H),
          ("bert.feed_forward_length", U32, F), ("bert.attention.head_count", U32, H // 32),
          ("bert.attention.layer_norm_epsilon", F32V, 1e-5), ("bert.context_length", U32, 64)]
    shapes = {"token_embd.weight": (8, H), "position_embd.weight": (64, H), "token_types.weight": (1, H),
              "token_embd_norm.weight": (H,), "token_embd_norm.bias": (H,)}
    for g, n in (("attn_q", H), ("attn_k", H), ("attn_v", H), ("attn_output", H), ("ffn_up", F), ("ffn_down", H)):
        shapes[f"blk.0.{g}.weight"] = (n, F if g == "ffn_down" else H)
        shapes[f"blk.0.{g}.bias"] = (n,)
    for g in ("attn_output_norm", "layer_output_norm"):
        shapes[f"blk.0.{g}.weight"] = shapes[f"blk.0.{g}.bias"] = (H,)
    tensors = []
    for name, shape in shapes.items():
        ty = linear_type if name.startswith("blk.") and len(shape) == 2 else F32
        rows, K = (shape if len(shape) == 2 else (1, shape[0]))
        tensors.append((name, ty, shape, random_blocks(ty, rows, K, rng).tobytes()))
    path = tmp_path / f"tiny-{H}-{linear_type}.gguf"
    write_gguf(path, md, tensors)
    return GGUFFile(path)


def test_plan_checks_quantized_linears(tmp_path) -> None:  # noqa: ANN001
    """A quantized linear whose K is not a multiple of 128 is refused by the plan, before any engine is built."""
    assert bert_plan(_tiny_bert(tmp_path, 128, 256, Q8_0)).hidden == 128
    assert bert_plan(_tiny_bert(tmp_path, 96, 192, F32)).hidden == 96
    with pytest.raises(ValueError, match="multiple of 128"):
        bert_plan(_tiny_bert(tmp_path, 96, 192, Q8_0))
