"""-m gpu: in-flight batching over a slot pool (engine.SlotPool, pipeline.run_slots / generate_continuous, Fo1ForCausalLM.generate_iter):
every request's tokens and length equal those of a static generate of n_slots sequences on the same decode path, bit for bit,
whatever its companions and whenever it was admitted; at <= 8 slots on the persistent kernel (<= 16 on the per-kernel path) those of
the request alone.  Slots are reused after longer and after shorter occupants; greedy and sampled requests mix; the refusals."""
import os
from importlib import import_module

import pytest
import torch

from tests.test_gpu_decode_mega import _engine

pytestmark = pytest.mark.gpu
MAX_NEW = (1, 3, 17, 40)


def _mods():
    import fo1_b200  # noqa: F401
    return import_module("vlm-fo1_b200.engine"), import_module("vlm-fo1_b200.pipeline")


@pytest.fixture(scope="module")
def eng():
    return _engine()[0]


def _requests(n, seed=0, n_short=0):
    """n requests: (embeddings bf16 [L, 2048], L, max_new_tokens), ragged prompt lengths.  The first n_short stop within 3 tokens, so
    that every slot of a pool that size takes a second request."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        L = 9 + (37 * i + 11 * seed) % 120
        m = MAX_NEW[i % 2] if i < n_short else MAX_NEW[(i * 3 + seed) % len(MAX_NEW)]
        out.append(((torch.randn(L, 2048, generator=g) * 0.05).bfloat16().cuda(), L, m))
    return out


def _pos(lens):
    return torch.cat([torch.arange(L, dtype=torch.int32).view(1, -1).expand(3, -1) for L in lens], 1).contiguous().cuda()


def _static(eng, reqs, T, stop, sampling=None):
    """One static Engine.generate over reqs with max_new_tokens T -> [(tokens, length)] per request, cut at its own limit."""
    lens = [L for _, L, _ in reqs]
    out = eng.generate(torch.cat([e for e, _, _ in reqs]), _pos(lens), lens, [0] * len(reqs), T, stop, 0, early_exit_interval=8,
                       sampling=sampling)
    res = []
    for b, (_, _, m) in enumerate(reqs):
        n = min(int(out["lens"][b]), m)
        res.append((out["tokens"][b, :n].clone(), n))
    return res


def _pool_run(eng, reqs, n_slots, stop, sampling=None):
    """reqs through a SlotPool of n_slots with the pipeline's host loop -> ({index: (tokens, length)}, {slot: [index, ...]})."""
    E, P = _mods()
    T = max(m for _, _, m in reqs)
    cap = max(L for _, L, _ in reqs) + T
    got, history = {}, {}
    with E.SlotPool(eng, n_slots, cap, T, stop, 0, sampled=sampling is not None) as pool:
        def admit(items, slots):
            lens = [reqs[i][1] for i in items]
            sp = None
            if sampling is not None:
                sp = E.Sampling(*([list(f)[i] for i in items] for f in (sampling.temperature, sampling.top_p, sampling.top_k, sampling.seed)))
            pool.admit(slots, torch.cat([reqs[i][0] for i in items]), _pos(lens), lens, torch.zeros(len(items), dtype=torch.int32, device="cuda"),
                       [reqs[i][2] for i in items], sampling=sp)
            for i, b in zip(items, slots):
                history.setdefault(b, []).append(i)
            return items

        def poll():
            return pool.finished.cpu().tolist(), pool.lens.cpu().tolist()
        for i, b, n in P.run_slots(len(reqs), n_slots, admit, pool.decode, poll):
            got[i] = (pool.tokens[b, :n].clone(), n)
    return got, history


def _stop_id(eng, reqs):
    """The 6th token of the request with the largest limit, alone: that request (at least) ends early on it."""
    i = max(range(len(reqs)), key=lambda j: reqs[j][2])
    return int(_static(eng, [reqs[i]], 40, [])[0][0][5])


def _assert_equal(got, want, reqs):
    assert sorted(got) == list(range(len(reqs)))
    for i, (t, n) in enumerate(want):
        gt, gn = got[i]
        assert gn == n and torch.equal(gt, t), (i, gn, n, gt.tolist(), t.tolist())


def _reuse(history, reqs, n_slots):
    """Every slot held at least two requests, and some slot followed a longer occupant with a shorter one and vice versa."""
    assert len(history) == n_slots and all(len(v) >= 2 for v in history.values()), history
    steps = lambda i: reqs[i][1] + reqs[i][2]
    pairs = [(a, b) for v in history.values() for a, b in zip(v, v[1:])]
    assert any(steps(a) > steps(b) for a, b in pairs) and any(steps(a) < steps(b) for a, b in pairs)


@pytest.mark.parametrize("no_mega,n_slots", [(False, 4), (True, 12)])
def test_pool_equals_each_request_alone(eng, monkeypatch, no_mega, n_slots):
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    reqs = _requests(11 if n_slots == 4 else 30, seed=n_slots, n_short=n_slots)
    stop = [_stop_id(eng, reqs)]
    got, history = _pool_run(eng, reqs, n_slots, stop)
    assert eng.last_decode_path() == (0 if no_mega else 1)
    want = [_static(eng, [r], r[2], stop)[0] for r in reqs]
    assert any(n < m for (_, n), (_, _, m) in zip(want, reqs)), "some request stops early"
    _assert_equal(got, want, reqs)
    _reuse(history, reqs, n_slots)


@pytest.mark.parametrize("no_mega,n_slots", [(False, 16), (True, 40)])
def test_pool_equals_static_batch_of_n_slots(eng, monkeypatch, no_mega, n_slots):
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    reqs = _requests(2 * n_slots, seed=n_slots)
    stop = [_stop_id(eng, reqs)]
    got, _ = _pool_run(eng, reqs, n_slots, stop)
    assert eng.last_decode_path() == (0 if no_mega else 1)
    want = _static(eng, reqs[:n_slots], 40, stop) + _static(eng, reqs[n_slots:], 40, stop)
    _assert_equal(got, want, reqs)


@pytest.mark.parametrize("no_mega", [False, True])
def test_pool_sampled_and_greedy_mixed(eng, monkeypatch, no_mega):
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    E, _ = _mods()
    n_slots = 4
    reqs = _requests(12, seed=7)
    greedy = [i % 3 == 2 for i in range(12)]
    samp = E.Sampling([1.0 if g else 0.8 for g in greedy], [1.0 if g else 0.9 for g in greedy], [1 if g else 40 for g in greedy],
                      [0 if g else 1000 + 17 * i for i, g in enumerate(greedy)])
    got, _ = _pool_run(eng, reqs, n_slots, [], sampling=samp)
    want = []
    for c in range(0, 12, n_slots):
        sub = E.Sampling(*(list(f)[c:c + n_slots] for f in (samp.temperature, samp.top_p, samp.top_k, samp.seed)))
        want += _static(eng, reqs[c:c + n_slots], 40, [], sampling=sub)
    _assert_equal(got, want, reqs)


def test_pool_refusals_and_guard(eng):
    E, _ = _mods()
    reqs = _requests(6, seed=3)
    stop = [_stop_id(eng, reqs)]
    ref, _ = _pool_run(eng, reqs, 2, stop)
    cap = max(L for _, L, _ in reqs) + 40
    F = import_module("vlm-fo1_b200._lib").Fo1Error
    with E.SlotPool(eng, 2, cap, 40, stop, 0) as pool:
        with pytest.raises(F):
            E.SlotPool(eng, 2, cap, 40, stop, 0)                          # one pool per model
        z = torch.zeros(1, dtype=torch.int32, device="cuda")
        e, L, m = reqs[0]
        for slots, lens, mnt, what in (([2], [L], [m], "out of range"), ([0], [cap], [m], "capacity"), ([0], [L], [41], "max_new")):
            with pytest.raises(F, match=what):
                pool.admit(slots, torch.cat([e] * (lens[0] // L + 1))[:lens[0]], _pos(lens), lens, z, mnt)
        pool.admit([0], e, _pos([L]), [L], z, [m])
        with pytest.raises(F, match="occupied"):
            pool.admit([0], e, _pos([L]), [L], z, [m])
        with pytest.raises(F, match="slot pool is open"):                # a plain generate must not touch the pool's cache
            eng.generate(e, _pos([L]), [L], [0], 4, stop, 0)
        pool.admit([1], reqs[1][0], _pos([reqs[1][1]]), [reqs[1][1]], z, [reqs[1][2]])
        pool.decode(0)
        for b in range(2):
            n = int(pool.lens[b])
            assert n == ref[b][1] and torch.equal(pool.tokens[b, :n], ref[b][0]), b
    out = eng.generate(e, _pos([L]), [L], [0], 4, stop, 0)                 # closed: generate runs again
    assert int(out["lens"][0]) >= 1


# ---------------------------------------------------------------------------------------------------------- Python surface
def test_generate_iter_and_refusals(fab_model, monkeypatch):
    model_path, model, kw = fab_model
    E, _ = _mods()
    # 11 requests on the six proposal-file images (mixed sizes and box counts; repeated images share the towers inside an admission
    # group) through 4 slots; the first four end within 3 tokens, so every slot takes a second request
    kws = [kw(i % 6, max_new=m) for i, m in enumerate((1, 3, 1, 3, 12, 6, 12, 2, 9, 12, 4))]
    history = {}
    admit = E.SlotPool.admit

    def recording(self, slots, inputs_embeds, position_ids, seq_lens, rope_deltas, max_new_tokens, sampling=None):
        for b, L, m in zip(slots, seq_lens, max_new_tokens):
            history.setdefault(b, []).append(int(L) + int(m))
        return admit(self, slots, inputs_embeds, position_ids, seq_lens, rope_deltas, max_new_tokens, sampling)
    monkeypatch.setattr(E.SlotPool, "admit", recording)
    got = dict(model.generate_iter(kws, batch_size=4))
    monkeypatch.setattr(E.SlotPool, "admit", admit)
    assert sorted(got) == list(range(len(kws)))
    assert len({k["images"][0].shape for k in kws}) > 1 and len({len(k["bbox_list"][0]) for k in kws}) > 1
    assert len(history) == 4 and all(len(v) >= 2 for v in history.values()), history
    pairs = [(a, b) for v in history.values() for a, b in zip(v, v[1:])]
    assert any(a > b for a, b in pairs) and any(a < b for a, b in pairs), history     # after a longer and after a shorter occupant
    for i, k in enumerate(kws):
        one = model.generate(**k)
        assert one.shape == got[i].shape and torch.equal(one, got[i].to(one.device)), (i, one.tolist(), got[i].tolist())
    # sampled and greedy mixed: seeds drawn in request order, as generate_batch draws them
    skws = [kw(i, temperature=0.7, top_p=0.9) for i in range(4)] + [kw(4)]
    torch.manual_seed(5)
    batch = model.generate_batch(skws)
    torch.manual_seed(5)
    got = dict(model.generate_iter(skws, batch_size=len(skws)))
    for i in range(len(skws)):
        assert torch.equal(batch[i], got[i].to(batch[i].device)), i
    a = kw(0)
    for name, bad in (("return_dict_in_generate", dict(return_dict_in_generate=True)), ("streamer", dict(streamer=object())), ("num_beams", dict(num_beams=2)),
                      ("prompt_lookup_num_tokens", dict(prompt_lookup_num_tokens=3)),
                      ("num_return_sequences", dict(num_return_sequences=2, do_sample=True, temperature=0.7)),
                      ("repetition_penalty", dict(do_sample=True, temperature=0.7, repetition_penalty=1.2))):
        k = dict(a, **bad)
        if name != "streamer":
            k["streamer"] = None
        with pytest.raises(NotImplementedError, match=name):
            list(model.generate_iter([k], batch_size=2))


@pytest.fixture(scope="module")
def fab_model(tmp_path_factory):
    import gzip
    import json
    from evaluation.common import ImageSource
    from vlm_fo1.mm_utils import prepare_inputs
    from vlm_fo1.model.builder import load_pretrained_model
    E, _ = _mods()
    FB = import_module("vlm-fo1_b200.fabricate")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    root = tmp_path_factory.mktemp("slots")
    cfg = E.EngineConfig()
    cfg.vit = dict(cfg.vit, depth=2, fullatt_block_indexes=[0, 1])
    cfg.davit = dict(cfg.davit, depths=[1, 1, 1, 1])
    cfg.llm = dict(cfg.llm, num_hidden_layers=1)
    model_path = FB.fabricate_checkpoint(str(root / "resources" / "VLM-FO1_Qwen2.5-VL-3B-v01"), cfg, seed=0, device="cuda")
    fx = json.load(gzip.open(os.path.join(repo, "tests", "golden", "eval_proposals_sample.json.gz"), "rt"))
    tokenizer, model, procs = load_pretrained_model(model_path, device="cuda:0")
    sizes = {im["file_name"]: (im["width"], im["height"]) for im in fx["instances"]["images"]}
    src = ImageSource(str(root / "none"), str(root / "synth"))
    msgs = []
    for d in fx["coco"][:6]:
        msgs.append([{"role": "user", "content": [{"type": "image_url", "image_url": {"url": src.path(d["image"], sizes[d["image"]])}},
                                                  {"type": "text", "text": d["conversations"][0]["value"]}], "bbox_list": d["bbox_list"]}])

    def kw(i, max_new=10, **k):
        k.setdefault("temperature", 0.0)
        k.setdefault("top_p", 0.05)
        return dict(prepare_inputs(model_path, model, procs, tokenizer, msgs[i], device="cuda:0", max_tokens=max_new, **k), streamer=None)
    return model_path, model, kw


def test_eval_coco_through_slots_equals_per_item_generate(tmp_path, monkeypatch):
    import gzip
    import json
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    E, _ = _mods()
    FB = import_module("vlm-fo1_b200.fabricate")
    from evaluation.eval_coco import eval_coco
    from vlm_fo1.model.fo1_model import Fo1ForCausalLM
    cfg = E.EngineConfig()
    cfg.vit = dict(cfg.vit, depth=2, fullatt_block_indexes=[0, 1])
    cfg.davit = dict(cfg.davit, depths=[1, 1, 1, 1])
    cfg.llm = dict(cfg.llm, num_hidden_layers=1)
    model_path = FB.fabricate_checkpoint(str(tmp_path / "resources" / "VLM-FO1_Qwen2.5-VL-3B-v01"), cfg, seed=0, device="cuda")
    fx = json.load(gzip.open(os.path.join(repo, "tests", "golden", "eval_proposals_sample.json.gz"), "rt"))
    with open(tmp_path / "coco.jsonl", "w") as f:
        for d in fx["coco"]:
            f.write(json.dumps(d) + "\n")
    json.dump(fx["instances"], open(tmp_path / "instances.json", "w"))
    # every answer becomes one prediction whose box depends on the answer's text, so the predictions file carries the tokens in item
    # order; the answers themselves are recorded too
    import zlib
    import evaluation.eval_coco as EC
    answers = []

    def extract(ans):
        answers.append(ans)
        return {"person": [zlib.crc32(ans.encode()) % 3]}
    monkeypatch.setattr(EC, "extract_predictions_to_indexes", extract)
    run = lambda out: eval_coco(model_path, str(tmp_path / "coco.jsonl"), str(tmp_path / "instances.json"), str(tmp_path / "none"),
                                out_dir=str(tmp_path / out), device="cuda:0", batch_size=4, limit=10, synthetic_images=str(tmp_path / "synth"),
                                max_tokens=12)
    monkeypatch.setattr(EC, "WINDOW", 1)           # windows of 4, 4 and 2 items: each through its own pool
    run("slots")
    slots_answers, answers[:] = list(answers), []

    def one_by_one(self, kwargs_iterable, batch_size=16, on_error=None):
        for i, k in enumerate(kwargs_iterable):
            yield i, self.generate(**k)
    monkeypatch.setattr(Fo1ForCausalLM, "generate_iter", one_by_one)
    run("single")
    assert len(slots_answers) == 10 and slots_answers == answers
    name = "VLM-FO1_Qwen2.5-VL-3B-v01/coco_predictions.json"
    res = json.load(open(tmp_path / "slots" / name))
    assert len(res) == 10 and [r["image_id"] for r in res] == [d["id"] for d in fx["coco"][:10]]
    assert (tmp_path / "slots" / name).read_bytes() == (tmp_path / "single" / name).read_bytes()
