"""AddressSanitizer + UndefinedBehaviorSanitizer and ThreadSanitizer builds of the host-only parts of the library (router,
tokenizer, JSON parser) driven by tests/native/host_sanitize.cc (SURVEY.md §5: race detection / memory checking on the path).  CPU only; skipped when g++ has no sanitizer runtime."""
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
SRC = [ROOT / "tests" / "native" / "host_sanitize.cc", ROOT / "kubeai_b200" / "csrc" / "router.cc", ROOT / "kubeai_b200" / "csrc" / "tokenizer.cc"]


def build(tmp_path, name, flags):
    if not shutil.which("g++"):
        pytest.skip("no g++")
    exe = tmp_path / name
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fno-omit-frame-pointer", *flags, *map(str, SRC), "-o", str(exe), "-lpthread"],
                       capture_output=True, text=True)
    if r.returncode != 0 and ("cannot find" in r.stderr or "unrecognized" in r.stderr):
        pytest.skip("sanitizer runtime not available: " + r.stderr.splitlines()[-1])
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def test_tokenizer_and_json_parser_under_asan_ubsan(tmp_path):
    tokenizers = pytest.importorskip("tokenizers")
    from tokenizers import Regex, Tokenizer, decoders, models, pre_tokenizers, trainers
    pat = r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+"
    tok = Tokenizer(models.BPE(ignore_merges=True))
    tok.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(pat), behavior="isolated"), pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    tok.decoder = decoders.ByteLevel()
    specials = ["<|begin_of_text|>", "<|end_of_text|>", "<|start_header_id|>", "<|end_header_id|>", "<|eot_id|>"]
    tok.train_from_iterator(["hello world it's 12345 naive cafe"] * 40, trainers.BpeTrainer(vocab_size=600, special_tokens=specials,
                            initial_alphabet=pre_tokenizers.ByteLevel.alphabet(), show_progress=False))
    path = tmp_path / "tokenizer.json"
    tok.save(str(path))
    exe = build(tmp_path, "host_asan", ["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"])
    r = subprocess.run([str(exe), "asan", str(path)], capture_output=True, text=True, timeout=600,
                       env={"ASAN_OPTIONS": "detect_leaks=1:abort_on_error=0", "UBSAN_OPTIONS": "print_stacktrace=1", "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and "asan leg ok" in r.stdout, (r.stdout[-500:], r.stderr[-3000:])
    assert "ERROR: AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr, r.stderr[-3000:]


def test_router_under_tsan(tmp_path):
    exe = build(tmp_path, "host_tsan", ["-fsanitize=thread"])
    r = subprocess.run([str(exe), "tsan"], capture_output=True, text=True, timeout=600, env={"TSAN_OPTIONS": "halt_on_error=0", "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and "tsan leg ok" in r.stdout, (r.stdout[-500:], r.stderr[-3000:])
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-3000:]
