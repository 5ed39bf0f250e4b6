"""CPU (no GPU): the float64 statement of the device sampler's contract (vitron_b200/sampling.py: Philox4x32-10, top-k /
top-p support sets), argument validation of vb200_sample_advance, and the host logic of sampled generate() on a CPU engine
(kernels replaced by tests/cpu_ops_emulator.py, the sampled step by the host statement)."""
import math
import os

import numpy as np
import pytest
import torch

from vitron_b200 import sampling as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("counter, key, want", [
    ([0, 0, 0, 0], [0, 0], "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0], "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(counter, key, want):
    """Random123's known-answer vectors for philox4x32-10."""
    got = E.philox4x32_10(np.array(counter), np.array(key))
    assert " ".join("%08x" % int(v) for v in got) == want


def direct_support(row, temperature, top_k, top_p):
    """The contract read literally, one token at a time (float64)."""
    z = [v / temperature for v in row]
    valid = [not math.isnan(v) for v in z]
    zv = sorted((v for v, ok in zip(z, valid) if ok), reverse=True)
    kept = list(valid)
    if 0 < top_k < len(zv):
        kept = [ok and v >= zv[top_k - 1] for v, ok in zip(z, kept)]
    zmax = zv[0]
    p = [(1.0 if v == zmax else math.exp(v - zmax)) if ok else 0.0 for v, ok in zip(z, kept)]
    if top_p < 1.0:
        tot = sum(p)
        kept = [ok and (sum(q for q, okj in zip(p, kept) if okj and q > p[i]) / tot < top_p or z[i] == zmax)
                for i, ok in enumerate(kept)]
    return kept


def test_support_sets_match_the_direct_definition():
    g = torch.Generator().manual_seed(0)
    rows = (torch.randint(-6, 6, (24, 40), generator=g).float() * 0.5)       # a half-integer grid: ties everywhere
    rows[3, 7] = float("nan")
    rows[5, :] = float("nan")
    rows[5, 11] = 0.25                                                        # one number in a row of NaNs
    rows[8, 2] = float("-inf")
    checked = 0
    for T in (0.5, 1.0, 3.0):
        for k in (0, 1, 3, 5, 40, 100):
            for p in (1.0, 0.0, 0.3, 0.5, 0.9):
                kept, probs, _ = E.sample_support(rows, T, k, p)
                for b in range(rows.shape[0]):
                    want = direct_support(rows[b].tolist(), T, k, p)
                    assert kept[b].tolist() == want, (T, k, p, b)
                    assert bool((probs[b][~kept[b]] == 0).all()) and bool((probs[b][kept[b]] >= 0).all())
                    checked += 1
    assert checked == 3 * 6 * 5 * 24


def test_ties_are_kept_together():
    row = torch.tensor([[3.0, 3.0, 1.0, 1.0, 1.0, 0.0, float("nan")]])
    kept, _, _ = E.sample_support(row, 1.0, 3, 1.0)                          # 3rd largest = 1.0: all three 1.0 stay
    assert kept[0].tolist() == [True] * 5 + [False, False]
    kept, _, _ = E.sample_support(row, 1.0, 0, 0.3)                          # both maxima stay (value-based top-p)
    assert kept[0].tolist() == [True, True] + [False] * 5
    kept, _, _ = E.sample_support(row, 1.0, 0, 0.0)                          # top_p = 0: the maximum always survives
    assert kept[0].tolist() == [True, True] + [False] * 5
    tok, _ = E.sample_reference(torch.full((2, 5), float("nan")), 1.0, 0, 1.0, 7, 0)
    assert tok.tolist() == [0, 0]                                             # no number in the row: token 0


def test_draw_follows_the_philox_stream():
    """top_k = 1 is the arg-max; with a flat row the draw is floor(u * V) of the stream's first word."""
    g = torch.Generator().manual_seed(1)
    lg = torch.randn((6, 50), generator=g)
    tok, _ = E.sample_reference(lg, 1.0, 1, 1.0, 123, 4)
    assert torch.equal(tok, lg.argmax(-1))
    flat = torch.zeros((6, 64))
    seed, step = 0x0123456789ABCDEF, 9
    tok, _ = E.sample_reference(flat, 1.0, 0, 1.0, seed, step)
    for b in range(6):
        x = int(E.philox4x32_10(np.array([step, b, 0, 0]), np.array([seed & 0xFFFFFFFF, seed >> 32]))[0])
        assert int(tok[b]) == (x >> 8) * 64 // 2 ** 24


@pytest.fixture(scope="module")
def lib():
    from vitron_b200 import _lib, build
    build.build()
    return _lib.load()


def test_sample_advance_argument_validation_without_device(lib):
    import ctypes as C
    buf = (C.c_uint8 * 4096)()
    p = C.addressof(buf)
    p += (-p) % 16
    ERR_ARG, ERR_UNSUP = -1, -4
    args = lambda logits=p, ld=8, rows=1, n=8, params=p, token_log=None, kv_len=None, prompt_len=None: (
        logits, ld, rows, n, params, p, None, None, kv_len, token_log, 8, prompt_len, None)
    assert lib.vb200_sample_advance(*args(logits=None)) == ERR_ARG
    assert lib.vb200_sample_advance(*args(params=None)) == ERR_ARG
    assert lib.vb200_sample_advance(*args(n=0)) == ERR_ARG
    assert lib.vb200_sample_advance(*args(n=-3)) == ERR_ARG
    assert lib.vb200_sample_advance(*args(rows=0)) == ERR_ARG
    assert lib.vb200_sample_advance(*args(ld=4)) == ERR_ARG                   # row stride shorter than a row
    assert lib.vb200_sample_advance(*args(token_log=p)) == ERR_ARG            # token_log needs kv_len and prompt_len
    assert lib.vb200_sample_advance(*args(n=1 << 20, ld=1 << 20)) == ERR_UNSUP  # row larger than shared memory


def tiny_model(monkeypatch):
    from oracle.weights import seeded_state_dict
    from vitron_b200.vision_tower import VisionConfig
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    from tests import cpu_ops_emulator
    cpu_ops_emulator.install(monkeypatch)
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "vitron_llm_tiny.pt"), weights_only=False)
    vit = dict(fx["vit"], hidden_act="gelu")
    cfg = VitronConfig(llm=fx["llm"], vision=VisionConfig(**vit), video=None, tokenizer_model_max_length=4096)
    model = VitronLlamaForCausalLM(cfg, "cpu", max_batch=2, max_seq_len=256)
    model.load_state_dict(seeded_state_dict(fx["shapes"], fx["seed"]))
    ids = torch.randint(3, fx["llm"]["vocab_size"], (2, 9), generator=torch.Generator().manual_seed(4))
    return model, ids


def test_sampled_generate_host_logic(monkeypatch):
    """generate(do_sample=True) on a CPU engine: top_k = 1 is greedy; the seed comes from torch's CPU
    generator, so one torch.manual_seed gives the same ids whatever the sync chunk; another seed gives other ids;
    EOS pads its row."""
    model, ids = tiny_model(monkeypatch)
    n = 7
    greedy = model.generate(ids, do_sample=False, max_new_tokens=n, eos_token_id=-1)
    assert torch.equal(model.generate(ids, do_sample=True, top_k=1, max_new_tokens=n, eos_token_id=-1), greedy)
    runs = []
    for seed, chunk in ((11, 16), (11, 3), (12, 16)):
        torch.manual_seed(seed)
        runs.append(model.generate(ids, do_sample=True, temperature=1.0, top_p=0.95, max_new_tokens=n, eos_token_id=-1,
                                   sync_every=chunk))
    assert runs[0].shape == (2, ids.shape[1] + n) and torch.equal(runs[0][:, :ids.shape[1]], ids)
    assert torch.equal(runs[0], runs[1])
    assert not torch.equal(runs[0], runs[2])
    eos = int(runs[0][0, ids.shape[1]])
    torch.manual_seed(11)
    got = model.generate(ids, do_sample=True, temperature=1.0, top_p=0.95, max_new_tokens=n, eos_token_id=eos, pad_token_id=0)
    assert int(got[0, ids.shape[1]]) == eos and bool((got[0, ids.shape[1] + 1:] == 0).all())
