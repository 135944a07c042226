"""The ordered event placement from block descriptors and two-entry output lists (k_blk_desc + k_expand_desc, option
expand_desc = 1) against the block-map walk (k_expand, expand_desc = 0), byte for byte: the batch shapes of
test_gpu_direct_events.py with the ordered placement forced, every Standard iterator, 2, 4 and 8 blocks in flight per
warp, lists of 255 and more, stream chunks, jobs, and a shard group whose second rank stages its tuples for the push
(the pad_like word offset)."""
import numpy as np
import pytest

import daachorse_b200 as D
from daachorse_b200 import synth as S

pytestmark = pytest.mark.gpu
MODES = (D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX)
# gather_ordered = 2: descriptors are made for the ordered placement only, which large batches get by default
DEFAULTS = {"kernel": 3, "event_queue": 0, "gather_ordered": 2, "expand_desc": 1, "expand_u": 2}


def _set(pma, **opts):
    for k, v in DEFAULTS.items():
        pma.set_option(k, opts.get(k, v))


def _batch(name, pool_bytes, n, n_patterns=None):
    import torch

    cfg = S.config(name)
    ps = S.make_patterns(cfg, n_patterns) if n_patterns else S.make_patterns(cfg)
    pool, b = S.make_pool(cfg, ps, pool_bytes)
    hay_len = cfg["hay_len"]
    starts = S.window_starts(b, len(pool), n, hay_len)
    text_t, offs_t = S.materialise_on_device(torch.from_numpy(pool).cuda(), torch.from_numpy(starts).cuda(), hay_len)
    return D.DoubleArrayAhoCorasick.new(ps.as_list()), text_t, offs_t


@pytest.mark.parametrize("name,pool_bytes,n", [("C2", 8 << 20, 4096), ("C3", 64 << 20, 16384)])
def test_descriptors_equal_block_map(name, pool_bytes, n):
    import torch

    pma, text_t, offs_t = _batch(name, pool_bytes, n)
    for mode in MODES:
        _set(pma, expand_desc=0)
        want = pma.scan_batch_device(mode, text_t, offs_t)
        assert want.matches.shape[0] > 0
        for queue in (0, 1):
            for u in (2, 4, 8):
                _set(pma, event_queue=queue, expand_u=u)
                r = pma.scan_batch_device(mode, text_t, offs_t)
                assert torch.equal(r.offsets, want.offsets), (name, mode, queue, u)
                assert torch.equal(r.matches, want.matches), (name, mode, queue, u)
    _set(pma)


@pytest.mark.parametrize("mode", MODES)
def test_long_lists_and_empty_pattern(mode):
    """`a` x k for k = 1..300 plus the empty pattern: lists of one, two, three and 255 or more in one batch, runs of
    tuples longer than a warp's staging buffer, and haystacks whose first tuple is at every word offset modulo 4."""
    import torch

    pats = [b""] + [b"a" * k for k in range(1, 301)] + [b"ba", b"b"]
    hays = [b"a" * 400, b"xa" + b"a" * 260 + b"b" + b"a" * 300, b"", b"ba" * 40, b"a" * 254, b"a" * 255, b"b", b"ab"]
    hays = hays * 40 + [b"a" * k for k in range(1, 70)]
    pma = D.DoubleArrayAhoCorasick.new(pats)
    text = np.frombuffer(b"".join(hays), dtype=np.uint8)
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    text_t, offs_t = torch.from_numpy(text.copy()).cuda(), torch.from_numpy(offs).cuda()
    for kernel in (0, 3):
        _set(pma, expand_desc=0)
        pma.set_option("kernel", kernel)
        want = pma.scan_batch_device(mode, text_t, offs_t)
        for u in (2, 4, 8):
            _set(pma, expand_u=u)
            pma.set_option("kernel", kernel)
            r = pma.scan_batch_device(mode, text_t, offs_t)
            assert torch.equal(r.offsets, want.offsets) and torch.equal(r.matches, want.matches), (kernel, u)
    _set(pma)


@pytest.mark.parametrize("mode", [D.FIND, D.FIND_OVERLAPPING])
def test_stream_chunks_descriptors_equal_block_map(mode):
    import torch

    cfg = S.config("C2")
    ps = S.make_patterns(cfg, n=4000)
    pool, _ = S.make_pool(cfg, ps, 4 << 20)
    rng = np.random.default_rng(37)
    n = 2000
    lens = rng.integers(0, 1200, size=n)
    starts = rng.integers(0, len(pool) - 1300, size=n)
    streams = [pool[int(s): int(s) + int(l)] for s, l in zip(starts, lens)]
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    states = {q: torch.zeros(n, dtype=torch.int32, device="cuda") for q in (0, 1)}
    pos = np.zeros(n, dtype=np.int64)
    while (pos < lens).any():
        k = rng.integers(0, 400, size=n)
        chunks = [st[int(p): int(p) + int(kk)] for st, p, kk in zip(streams, pos, k)]
        offs = np.zeros(n + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(c) for c in chunks])
        text = np.concatenate(chunks) if offs[-1] else np.zeros(0, np.uint8)
        t = torch.from_numpy(np.ascontiguousarray(text)).cuda() if len(text) else torch.zeros(16, dtype=torch.uint8, device="cuda")[:0]
        o = torch.from_numpy(offs).cuda()
        p = torch.from_numpy(pos.astype(np.int32)).cuda()
        got = {}
        for q in (0, 1):
            _set(pma, expand_desc=q)
            got[q] = pma.scan_stream_device(mode, t, o, states[q], p)
        assert torch.equal(got[0].offsets, got[1].offsets) and torch.equal(got[0].matches, got[1].matches)
        assert torch.equal(states[0], states[1])
        pos += np.array([len(c) for c in chunks])
    _set(pma)


def test_jobs_descriptors_equal_block_map():
    import torch

    pma, text_t, offs_t = _batch("C3", 16 << 20, 4096, n_patterns=60000)
    dev = torch.device("cuda", 0)
    half = (offs_t.numel() - 1) // 2
    parts = [(text_t, offs_t[: half + 1]), (text_t, offs_t[half:])]
    _set(pma, expand_desc=0)
    want = [pma.scan_batch_device(D.FIND_OVERLAPPING, tt, oo) for tt, oo in parts]
    _set(pma)
    streams = [torch.cuda.Stream(dev) for _ in range(2)]
    jobs = [pma.job(0), pma.job(0)]
    caps = [want[0].matches.shape[0] + 7, want[1].matches.shape[0]]  # slack, and the exact size
    outs = [torch.zeros((c, 3), dtype=torch.int32, device=dev) for c in caps]
    oofs = [torch.zeros(p[1].numel(), dtype=torch.int64, device=dev) for p in parts]
    torch.cuda.synchronize()
    for _ in range(2):
        for k in range(2):
            jobs[k].scan(D.FIND_OVERLAPPING, parts[k][0], parts[k][1], outs[k].shape[0], stream=streams[k])
        for k in range(2):
            jobs[k].place(outs[k], oofs[k], stream=streams[k])
        for k in range(2):
            assert jobs[k].wait() == want[k].matches.shape[0]
            assert torch.equal(outs[k][: want[k].matches.shape[0]], want[k].matches)
            assert torch.equal(oofs[k], want[k].offsets)


@pytest.mark.parametrize("world", [2, 3])
def test_shard_group_descriptors_equal_block_map(world):
    import torch

    from daachorse_b200 import shard

    pma, text_t, offs_t = _batch("C3", 16 << 20, 1536, n_patterns=60000)
    text, offs = text_t.cpu().numpy(), offs_t.cpu().numpy().astype(np.uint64)
    n = len(offs) - 1
    _set(pma, expand_desc=0)
    whole = pma.scan_batch_device(D.FIND_OVERLAPPING, text_t, offs_t)
    _set(pma)
    bounds = shard.byte_balanced_ranges(offs, world)
    cap = int(whole.matches.shape[0]) + 64
    groups = [shard.PeerGroup(r, world, 0, cap, n, exchange=None) for r in range(world)]
    blobs = [g.handle for g in groups]
    for g in groups:
        g.connect(blobs)
    jobs = [pma.job(0) for _ in range(world)]
    streams = [torch.cuda.Stream(torch.device("cuda", 0)) for _ in range(world)]
    inputs = []
    for r in range(world):
        lo, hi = bounds[r], bounds[r + 1]
        inputs.append((torch.from_numpy(text[int(offs[lo]): int(offs[hi])]).cuda(),
                       torch.from_numpy((offs[lo: hi + 1] - offs[lo]).astype(np.int64)).cuda()))
    for r in range(world):
        jobs[r].scan(D.FIND_OVERLAPPING, inputs[r][0], inputs[r][1], cap, stream=streams[r])
    for r in range(world):
        groups[r].place(jobs[r], bounds[r], r == world - 1, stream=streams[r])
    for r in reversed(range(1, world)):
        groups[r].finish(stream=streams[r])
    total = groups[0].finish(stream=streams[0])
    m, o = groups[0].result(total)
    assert total == whole.matches.shape[0]
    assert torch.equal(m, whole.matches) and torch.equal(o, whole.offsets)
    for g in groups:
        g.close()
