"""Encoding to a target quality (Encoder.set_target_mse / set_target_psnr; openjph_b200/csrc/rate_ctrl.cu).

Each configuration is encoded at four targets, from near-lossless to one that leaves most code-blocks out.  Every stream
must:
  * decode (library Decoder) to samples whose squared error against the source, in Python integers, equals the 128-bit
    SSE quality_info reports, and is at most floor(target * N) whenever the target was reached;
  * decode with the unmodified reference: 5/3 samples equal ours, 9/7 samples at most 1 apart inside the tie band;
  * carry, for every included block, the missing-MSB count K_max - 1 - k, the cleanup length R_b(k) and the bytes the
    reference block encoder writes at those missing MSBs;
  * end with a closed bracket, reached by the search rule restated here (search_replay) over the reported rounds: the
    model's proposals (summed in the device's order, so bit for bit), the correction factor, the halving rounds.
Edges, paths (host planes, resident graph replays, tensors), launch counts and refusals follow.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

import cases
import ratemodel
from openjph_b200 import codestream as cs
from test_rate_control import CPU_CONFIGS as _RC, _block_words, _decode_ours

FULL = 1 << 32
MODEL_ROUNDS, BODY_ROUNDS = 4, 16          # RQ_MODEL_ROUNDS, RQ_BODY_ROUNDS of ojb_device.h
RS_THREADS = 1024                          # the select kernel's CTA (rate_ctrl.cu)

_BY_NAME = dict(_RC)
CPU_CONFIGS = [(n, _BY_NAME[n]) for n in ("rev_rct", "irv_ict_q90", "irv_gray_qstep", "rev_signed10", "rev_sub420",
                                          "dfs_atk_irv", "tiles_tp_tlm_off", "prec_RPCL", "prec_CPRL")] + [
    ("nlt_irv_ict", dict(width=120, height=90, num_comps=3, bit_depth=10, is_signed=True, num_decomps=3, reversible=False,
                         color_transform=True, qstep=0.002, nlt={"all": 3})),
    # zero decomposition levels: blocks that may lose a sample (ENC_CHECK_NEGZERO), so key 0 is measured, not assumed
    ("rev_gray_L0", dict(width=64, height=64, num_comps=1, bit_depth=8, num_decomps=0, reversible=True)),
]
GPU_CONFIGS = [
    ("hd_rev_rct", dict(width=1920, height=1080, num_comps=3, bit_depth=8, num_decomps=5, reversible=True, color_transform=True)),
    ("4k_irv_q90", dict(width=4096, height=4096, num_comps=3, bit_depth=12, num_decomps=5, reversible=False, color_transform=True, qfactor=90)),
    ("8k_rev_rct", dict(width=8192, height=8192, num_comps=3, bit_depth=12, num_decomps=5, reversible=True, color_transform=True)),
]


def sse_of(planes, frame):
    return sum(int(np.sum((a.astype(np.int64) - f.astype(np.int64)) ** 2, dtype=np.int64)) if a.size < (1 << 20) else
               sum(int(np.sum((a[i:i + 256].astype(np.int64) - f[i:i + 256].astype(np.int64)) ** 2, dtype=np.int64))
                   for i in range(0, a.shape[0], 256))
               for a, f in zip(planes, frame))


def limit_of(mse, n):
    return math.floor(Fraction(mse) * n)


def lossless0_of(p):
    """the unconstrained selection is known to decode to the source (the device's rq_lossless0): every component is
    reversible and none has zero decomposition levels (whose blocks carry ENC_CHECK_NEGZERO and may lose a sample)"""
    for c in range(p.num_comps):
        rev = p.coc_reversible[c] if p.coc_present[c] else p.reversible
        nd = p.coc_num_decomps[c] if p.coc_present[c] else p.num_decomps
        if not rev or nd == 0:
            return False
    return True


class Body:
    """sum_b R_b(k_b(t)) and sum_b D_b(k_b(t)) restated from the device's own tables (rate_info); key 0 is the
    unconstrained selection"""
    def __init__(self, info):
        kmax, R = info["kmax"].astype(int), info["R"]
        self.D = info["D"]
        self.hulls = [ratemodel.hull(R[b], info["D"][b], int(kmax[b])) for b in range(len(kmax))]
        self.sum0 = sum(int(R[b][0]) for b in range(len(kmax)) if kmax[b] > 0 and R[b][0] != ratemodel.INVALID)

    def dist(self, t):
        """in the select kernel's order: thread b % RS_THREADS sums its blocks in index order, then a fixed tree"""
        part = np.zeros(RS_THREADS)
        for b, (ks, keys, lens) in enumerate(self.hulls):
            k = 0 if t == 0 else ks[ratemodel.taken(keys, t)]
            part[b % RS_THREADS] += self.D[b][k]
        d = RS_THREADS // 2
        while d:
            part[:d] += part[d:2 * d]
            d >>= 1
        return float(part[0])

    def model(self, c, limit):
        """the largest key whose modelled error is within c * limit (0 when none is)"""
        lim = c * float(limit)
        if self.dist(FULL) <= lim:
            return FULL
        if not self.dist(0) <= lim:
            return 0
        lo, hi = 0, FULL
        while hi - lo > 1:
            mid = (lo + hi) >> 1
            if self.dist(mid) <= lim:
                lo = mid
            else:
                hi = mid
        return lo

    def __call__(self, t):
        if t == 0:
            return self.sum0
        s = 0
        for ks, keys, lens in self.hulls:
            j = ratemodel.taken(keys, t)
            s += lens[j - 1] if j else 0
        return s

    def fitting(self, budget):
        if self(0) <= budget:
            return 0
        lo, hi = 0, FULL
        while hi - lo > 1:
            mid = (lo + hi) >> 1
            if self(mid) <= budget:
                hi = mid
            else:
                lo = mid
        return hi


def search_replay(q, lossless0, body=None):
    """the search rule over the reported rounds: every key lies inside the bracket of its round and follows the rule
    of that round; the bracket closes exactly after the last round.  body: restated bodies (checks every round's body
    and the halving rounds' keys; None on frames too large to restate)"""
    tp, tf, bp, bf = 0, FULL, q["body0"], 0
    if body is not None:
        assert body(0) == bp
    passed, failed, state = lossless0, False, {"done": False, "zero": False}
    limit, c = q["limit"], 1.0

    def close():
        if tf - tp <= 1 or (bp - bf) * 400 <= bp or bp - bf <= 64:
            state["done" if passed else "zero"] = True

    close()
    for r, rd in enumerate(q["rounds"]):
        assert not state["done"], r
        key = rd["key"]
        if body is not None:
            assert rd["body"] == body(key), (r, key)
        if state["zero"]:
            assert key == 0, r
        elif r < MODEL_ROUNDS and body is not None:
            tm = body.model(c, limit)
            if (tp < tm < tf) or (tm == FULL and not failed):
                want = tm
            elif tm <= tp:
                want = tp + 1
            else:
                want = min(max(body.fitting((bp + bf) >> 1), tp + 1), tf - 1)
            assert key == want, (r, key, want, tm, tp, tf)
            if r == 0:
                assert q["model_round1"] == body.dist(key)
        elif r < MODEL_ROUNDS:
            assert (tp < key < tf) or (key == FULL and not failed), (r, key, tp, tf)
        elif r < BODY_ROUNDS:
            if body is not None:
                assert key == min(max(body.fitting((bp + bf) >> 1), tp + 1), tf - 1), (r, key)
            assert tp < key < tf, (r, key, tp, tf)
        else:
            assert key == (tp + tf) >> 1, (r, key)
        ok = rd["sse"] <= limit
        if ok or key == 0:
            tp, bp, passed = key, rd["body"], True
            if not ok:
                state["done"] = True
                continue
        else:
            tf, bf, failed = key, rd["body"], True
        s = float(rd["sse"] >> 64) * 18446744073709551616.0 + float(rd["sse"] & ((1 << 64) - 1))
        c = c * float(limit) / s if s > 0 else c * 2.0
        close()
    assert state["done"], "the bracket did not close"
    assert (q["pass_key"], q["fail_key"], q["pass_body"], q["fail_body"]) == (tp, tf, bp, bf)
    assert q["fail_measured"] == failed
    if failed:
        assert [rd["sse"] for rd in q["rounds"] if rd["key"] == tf][-1] > limit


def check_stream(L, ref, p, frame, enc, j2c, mse, blocks_check=True, byte_sample=40, lossless0=None):
    q = enc.quality_info()
    n = sum(int(np.asarray(f).size) for f in frame)
    assert q["num_samples"] == n and q["limit"] == limit_of(mse, n)
    ours, blocks = _decode_ours(L, j2c)
    assert sse_of(ours, frame) == q["sse"], "the reported squared error is not the decoded one"
    if q["reached"]:
        assert q["sse"] <= q["limit"]
    assert abs(sum(q["comp_sse"]) - q["sse"]) <= 1e-9 * max(1, q["sse"])
    rev = bool(p.reversible)
    if lossless0 is None:
        lossless0 = lossless0_of(p)
    if blocks_check:
        info = enc.rate_info()
        kmax, k, R = info["kmax"].astype(int), info["k"].astype(int), info["R"]
        assert len(blocks) == len(k)
        for b, bd in enumerate(blocks):
            if k[b] < kmax[b] and R[b][k[b]]:
                assert bd.missing_msbs == kmax[b] - 1 - k[b] and bd.len1 == R[b][k[b]], b
            else:
                assert bd.len1 == 0, b
        words = _block_words(enc, p, blocks)
        inc = [b for b, bd in enumerate(blocks) if bd.len1]
        if len(inc) > byte_sample:
            inc = sorted(np.random.default_rng(5).choice(inc, size=byte_sample, replace=False).tolist())
        for b in inc:
            bd = blocks[b]
            assert j2c[bd.byte_off:bd.byte_off + bd.len1] == ref.encode_block(np.ascontiguousarray(words[b], np.uint32),
                                                                              int(bd.missing_msbs)), b
        search_replay(q, lossless0, Body(info))
    else:
        search_replay(q, lossless0)
    theirs, _ = ref.decode(j2c)
    if rev:
        for a, r_ in zip(ours, theirs):
            assert np.array_equal(a, r_)
    else:
        cases.assert_irv_matches_reference(ours, theirs, "quality", list(p.bit_depth)[:p.num_comps])
    return q, ours


def _mse(planes, frame):
    return sse_of(planes, frame) / sum(int(np.asarray(f).size) for f in frame)


def _targets(L, p, frame):
    """near-lossless (or just above the 9/7 floor) up to a target that leaves most blocks out"""
    full = cs.Encoder(p, lib=L).encode(frame)
    floor = _mse(_decode_ours(L, full)[0], frame)
    e = cs.Encoder(p, lib=L, target_bytes=cs.Encoder(p, lib=L).min_size)
    empty = _mse(_decode_ours(L, e.encode(frame))[0], frame)
    lo = max(floor * 1.5, empty * 1e-4, 0.05)
    hi = empty * 0.6
    return full, floor, empty, [lo * (hi / lo) ** (i / 3) for i in range(4)]


def _run_config(L, ref, name, kw):
    p = cases.make(kw)
    frame = cases.frame_for(p)
    full, floor, empty, targets = _targets(L, p, frame)
    enc = cs.Encoder(p, lib=L)
    for mse in targets:
        enc.set_target_mse(mse)
        j2c = enc.encode(frame)
        q, _ = check_stream(L, ref, p, frame, enc, j2c, mse)
        assert q["reached"], (name, mse)
        assert len(j2c) <= len(full) + 64
    enc.close()


@pytest.mark.parametrize("name,kw", CPU_CONFIGS, ids=[c[0] for c in CPU_CONFIGS])
def test_quality_target_emulator(emu_lib, ref, name, kw):
    _run_config(emu_lib, ref, name, kw)


def _edge_checks(L, ref):
    # reversible, a target below any loss: the unconstrained bytes
    p = cases.make(_BY_NAME["rev_rct"])
    frame = cases.frame_for(p)
    full = cs.Encoder(p, lib=L).encode(frame)
    e = cs.Encoder(p, lib=L, target_mse=1e-9)
    j = e.encode(frame)
    assert j == full and e.quality_info()["sse"] == 0 and e.quality_info()["reached"]
    # above the error of the empty stream: the min_size stream
    _, _, empty, _ = _targets(L, p, frame)
    e = cs.Encoder(p, lib=L, target_mse=empty * 10)
    j = e.encode(frame)
    assert len(j) == e.min_size
    check_stream(L, ref, p, frame, e, j, empty * 10, byte_sample=0)
    # deterministic
    e2 = cs.Encoder(p, lib=L, target_mse=empty * 0.01)
    assert e2.encode(frame) == e2.encode(frame) == cs.Encoder(p, lib=L, target_mse=empty * 0.01).encode(frame)
    # irreversible, below the quantisation floor: the unconstrained stream, not reached
    p = cases.make(_BY_NAME["irv_ict_q90"])
    frame = cases.frame_for(p)
    full = cs.Encoder(p, lib=L).encode(frame)
    floor = _mse(_decode_ours(L, full)[0], frame)
    e = cs.Encoder(p, lib=L, target_mse=floor * 0.5)
    j = e.encode(frame)
    q, _ = check_stream(L, ref, p, frame, e, j, floor * 0.5, byte_sample=0)
    assert j == full and not q["reached"] and q["sse"] > q["limit"]
    # PSNR: peak 2^B - 1
    e = cs.Encoder(p, lib=L, target_psnr=30.0)
    j = e.encode(frame)
    q = e.quality_info()
    assert q["limit"] == limit_of(4095.0 ** 2 / 10.0 ** 3.0, q["num_samples"])
    assert q["reached"] and 10 * math.log10(4095.0 ** 2 * q["num_samples"] / max(1, q["sse"])) >= 30.0


def test_quality_target_edges_emulator(emu_lib, ref):
    _edge_checks(emu_lib, ref)


def _path_checks(L, kw, mse):
    """host planes, the resident form (eager, captured, replayed) and target 0: bytes and launches"""
    p = cases.make(kw)
    frames = [cases.frame_for(p, seed=s) for s in (1, 2, 3)]
    single = [cs.Encoder(p, lib=L, target_mse=mse).encode(f) for f in frames]
    e = cs.Encoder(p, lib=L, target_mse=mse)
    for f, want in zip(frames, single):
        e.upload(f)
        assert e.encode_resident() == want
    plain = cs.Encoder(p, lib=L)
    want = plain.encode(frames[0])
    e.set_target_mse(0)
    assert e.encode(frames[0]) == want and e.kernel_launches == plain.kernel_launches
    return p, frames, single


def test_quality_target_paths_emulator(emu_lib):
    _path_checks(emu_lib, _BY_NAME["rev_rct"], 2.0)
    _path_checks(emu_lib, _BY_NAME["irv_ict_q90"], 20000.0)


def _refusal_checks(L):
    import ctypes as C
    p = cases.make(dict(width=64, height=64, num_comps=1, bit_depth=8, num_decomps=2, reversible=True))
    e = cs.Encoder(p, lib=L)
    with pytest.raises(cs.OjphError, match="0x000B004B"):
        e.quality_info()
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(cs.OjphError, match="0x000B0048"):
            e.set_target_mse(bad)
    e.set_target_size(e.min_size + 100)
    with pytest.raises(cs.OjphError, match="0x000B0049"):
        e.set_target_mse(1.0)
    e.set_target_size(0)
    e.set_target_mse(1.0)
    with pytest.raises(cs.OjphError, match="0x000B0049"):
        e.set_target_size(e.min_size + 100)
    e.encode(cases.frame_for(p))
    # a reconfigure to a configuration the target cannot serve: the next frame call refuses
    pe = cases.make(dict(width=1, height=2, num_comps=2, bit_depth=8, num_decomps=2, reversible=True, prog_order="RLCP",
                         tilepart_div=1, offset=(0, 1)))
    assert e.L.ojb_enc_configure(e.h, C.byref(pe), cs.I32) == 0
    e.params, e.dims = pe, cs.comp_dims(pe)
    with pytest.raises(cs.OjphError, match="0x000B004A"):
        e.encode(cases.frame_for(pe))
    e.close()
    e = cs.Encoder(pe, lib=L)
    with pytest.raises(cs.OjphError, match="0x000B004A"):
        e.set_target_mse(1.0)
    e.close()
    pw = cs.make_params(64, 64, 3, 32, num_decomps=5, reversible=True, color_transform=True)
    e = cs.Encoder(pw, lib=L)
    with pytest.raises(cs.OjphError, match="0x000B004A"):
        e.set_target_mse(1.0)
    e.close()
    pm = cases.make(dict(width=64, height=64, num_comps=2, bit_depth=8, num_decomps=2, reversible=True))
    pm.bit_depth[1] = 10
    e = cs.Encoder(pm, lib=L)
    with pytest.raises(ValueError):
        e.set_target_psnr(40.0)
    e.close()


def test_quality_target_refusals_emulator(emu_lib):
    _refusal_checks(emu_lib)


# ---- on the H100 -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", CPU_CONFIGS, ids=[c[0] for c in CPU_CONFIGS])
def test_quality_target_gpu_small(gpu_lib, ref, name, kw):
    _run_config(gpu_lib, ref, name, kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", GPU_CONFIGS, ids=[c[0] for c in GPU_CONFIGS])
def test_quality_target_gpu_large(gpu_lib, ref, name, kw):
    p = cases.make(kw)
    frame = cases.frame_for(p)
    if p.reversible:
        targets = (40.0, 45.0, 50.0) if kw["bit_depth"] >= 12 else (32.0, 38.0, 44.0)
    else:
        # under the quantisation floor (about 36.2 dB for the 4K q90 frame) every target ends on the floor path: the
        # targets sit below the measured floor, so each is a real search that must reach its target
        peak = float((1 << int(p.bit_depth[0])) - 1)
        floor = _mse(_decode_ours(gpu_lib, cs.Encoder(p, lib=gpu_lib).encode(frame))[0], frame)
        floor_db = 10.0 * math.log10(peak * peak / floor)
        targets = (floor_db - 0.75, floor_db - 3.0, floor_db - 6.0)
    enc = cs.Encoder(p, lib=gpu_lib)
    for db in targets:
        enc.set_target_psnr(db)
        j2c = enc.encode(frame)
        q, _ = check_stream(gpu_lib, ref, p, frame, enc, j2c, enc_mse(p, db), blocks_check=False)
        assert q["reached"] and q["pass_key"] > 0, (name, db, q["pass_key"])
    enc.close()


def enc_mse(p, db):
    peak = float((1 << int(p.bit_depth[0])) - 1)
    return peak * peak / 10.0 ** (db / 10.0)


@pytest.mark.gpu
def test_quality_target_edges_gpu(gpu_lib, ref):
    _edge_checks(gpu_lib, ref)


@pytest.mark.gpu
def test_quality_target_refusals_gpu(gpu_lib):
    _refusal_checks(gpu_lib)


@pytest.mark.gpu
@pytest.mark.parametrize("name,mse", [("rev_rct", 2.0), ("irv_ict_q90", 20000.0)])
def test_quality_target_paths_gpu(gpu_lib, name, mse):
    import torch
    p, frames, single = _path_checks(gpu_lib, _BY_NAME[name], mse)
    e = cs.Encoder(p, lib=gpu_lib, target_mse=mse)
    for f, want in zip(frames, single):
        chw = torch.from_numpy(np.stack(f)).cuda()
        assert bytes(e.encode_tensor(chw, "chw").cpu().numpy()) == want
        hwc = chw.permute(1, 2, 0).contiguous()
        assert bytes(e.encode_tensor(hwc, "hwc").cpu().numpy()) == want
