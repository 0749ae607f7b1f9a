"""CPU: every scratch layout the engine carves, through lg_test_scratch_regions, for c2i and t2i models in f32, bf16 and fp16 (and an
fp8 KV cache), head dims 64, 100 and 128, odd rows and sequence lengths, CFG on and off, SJD windows of 2 and 16 and a given array with
LEAD, EXTEND and TAIL segments.

Every layout: regions 256-byte aligned and pairwise disjoint, the last one ending within 255 bytes of what the kind's *_workspace_bytes
reports, and exactly the expected regions holding int state (tokens, counters, the window's tokens and positions, the SJD ints, the
uploaded given tokens) or KV cache. The two-chain view of the workspace: each chain's part of a region that scales with rows is exactly
its half of the full region, the two chains' GEMM partial slices are disjoint, 64-float aligned and each large enough for a chain's own
rows, and chain g's loop counters and sampler ticket lie inside the counter region."""
import ctypes
import itertools

import numpy as np
import pytest

from llamagen_b200 import _lib

WS, SCORE, PREFIX, SLOT, SLOT_PREFIX, SLOT_EXTEND, GIVEN, SJD, SJD_SLOTS = range(9)
DATA, INT, KV = 0, 1, 2
ROWS = [DATA] * 8                                  # carve_rows: h, xn, q, attn, ff, x0, partial, logits
PARTIAL = 6                                        # index of the GEMM partials in ROWS
KV_PAIR = [KV, KV]
COUNTER_INTS, TICKET = 128, 64                     # kCounterInts; chain g's ticket is counter 64 + 2g
GIVEN_LEN = 17                                     # LEAD [0, 4), EXTEND 8..10, TAIL 14..16 of an image of 17 tokens


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def _lib_or_skip():
    try:
        return _lib.load()
    except Exception as exc:   # pragma: no cover - the library is built by build()
        pytest.skip(f"libllamagen_b200 not built: {exc}")


def _engine(lib, model_type, dtype, hd, kv_f8=False):
    n_head = 2
    dim = n_head * hd
    tc = 1 if model_type == _lib.LG_MODEL_C2I else 7
    cfg = _lib.ModelCfg(2, n_head, dim, 3 * dim - 8 if dim % 16 == 8 else 3 * dim, 1000, tc, 48, 10, 72, model_type, dtype, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0, lib.lg_last_error()
    if kv_f8:
        assert lib.lg_engine_set_kv_cache(h, _lib.LG_DTYPE_E4M3, None) == 0, lib.lg_last_error()
    return h, cfg


def _regions(lib, h, kind, args, given=None):
    a = np.asarray(args, np.int64)
    n = lib.lg_test_scratch_regions(h, kind, _p(a), len(a), None if given is None else _p(given), None, 0)
    assert n > 0, lib.lg_last_error()
    out = np.zeros((n, 4), np.int64)
    assert lib.lg_test_scratch_regions(h, kind, _p(a), len(a), None if given is None else _p(given), _p(out), n) == n
    return out


def _bytes(lib, fn, *args):
    n = ctypes.c_size_t()
    assert getattr(lib, fn)(*args, ctypes.byref(n)) == 0, lib.lg_last_error()
    return n.value


def _check(regs, size, classes, tight=True):
    """Aligned, disjoint, within `size`, ending within 255 bytes of it (tight) and classed as `classes`."""
    assert regs[:, 2].tolist() == classes
    assert (regs[:, 0] % 256 == 0).all() and (regs[:, 1] >= 0).all()
    live = regs[regs[:, 1] > 0]
    order = live[np.argsort(live[:, 0], kind="stable")]
    assert (order[1:, 0] >= order[:-1, 0] + order[:-1, 1]).all(), "overlapping regions"
    end = int((regs[:, 0] + regs[:, 1]).max())
    assert end <= size and (not tight or size - end <= 255), (end, size)
    assert int(regs[-1, 0] + regs[-1, 1]) == end   # carving order is address order


def _given():
    g = np.full((3, GIVEN_LEN), -1, np.int32)
    g[:, :4] = [[5, 6, 7, 8]] * 3
    g[:, 8:11] = 9
    g[:, 14:] = 11
    return g


CONFIGS = [(mt, dt, hd, False) for mt, dt, hd in itertools.product(
    (_lib.LG_MODEL_C2I, _lib.LG_MODEL_T2I), (_lib.LG_DTYPE_F32, _lib.LG_DTYPE_BF16, _lib.LG_DTYPE_F16), (64, 100, 128))]
CONFIGS += [(mt, _lib.LG_DTYPE_BF16, hd, True) for mt in (_lib.LG_MODEL_C2I, _lib.LG_MODEL_T2I) for hd in (64, 100)]
CONFIGS += [(_lib.LG_MODEL_T2I, _lib.LG_DTYPE_F16, 128, True)]


def _cid(c):
    return f"{'c2i' if c[0] == _lib.LG_MODEL_C2I else 't2i'}-{['f32', 'bf16', 'fp16'][c[1]]}-hd{c[2]}{'-kv8' if c[3] else ''}"


@pytest.mark.parametrize("conf", CONFIGS, ids=_cid)
def test_every_layout_is_aligned_disjoint_and_classed(conf):
    lib = _lib_or_skip()
    h, cfg = _engine(lib, *conf)
    tc, t2i = cfg.cls_token_num, conf[0] == _lib.LG_MODEL_T2I
    try:
        for rows, seq in [(3, tc + 5), (6, tc + 16), (1, tc + 1), (33, 47)]:
            _check(_regions(lib, h, WS, [rows, seq]), _bytes(lib, "lg_engine_workspace_bytes", h, rows, seq),
                   KV_PAIR + ROWS + [INT, INT])
        for rows, seq in [(1, tc), (3, tc + 1), (4, tc + 8), (5, tc + 13), (2, tc + 47)]:
            _check(_regions(lib, h, SCORE, [rows, seq]), _bytes(lib, "lg_score_workspace_bytes", h, rows, seq), KV_PAIR + ROWS)
            _check(_regions(lib, h, PREFIX, [rows, seq]), _bytes(lib, "lg_prefix_workspace_bytes", h, rows, seq), ROWS)
        for cfg_on in (0, 1):
            if t2i:
                _check(_regions(lib, h, SLOT, [cfg_on]), _bytes(lib, "lg_slot_workspace_bytes", h, cfg_on), ROWS + [DATA, DATA])
            for P in (0, 1, 9, 47):
                _check(_regions(lib, h, SLOT_PREFIX, [cfg_on, P]), _bytes(lib, "lg_slot_prefix_workspace_bytes", h, cfg_on, P),
                       ROWS + [DATA, DATA])
            for K in (1, 5, 46):
                _check(_regions(lib, h, SLOT_EXTEND, [cfg_on, K]), _bytes(lib, "lg_slot_extend_workspace_bytes", h, cfg_on, K),
                       ROWS + [INT, INT, DATA, DATA])
            for B, L in [(1, 2), (3, 16), (5, 2), (4, 16)]:
                sjd = ROWS + [DATA, DATA] + [INT] * 10     # p, q, then seed_rows .. state
                _check(_regions(lib, h, SJD, [B, cfg_on, L]), _bytes(lib, "lg_sjd_workspace_bytes", h, B, cfg_on, L), sjd)
                _check(_regions(lib, h, SJD_SLOTS, [B, cfg_on, L]), _bytes(lib, "lg_sjd_slots_workspace_bytes", h, B, cfg_on, L),
                       sjd + [INT, INT, DATA, INT, INT])          # seed_slots, pass_slots, cfg_rows, interval_rows, img_slots
            for g, n_chain in [(_given(), 1), (_given()[:2], 2), (np.where(_given()[:2] >= 0, -1, 0).astype(np.int32), 2)]:
                B = g.shape[0]
                size = _bytes(lib, "lg_given_workspace_bytes", h, _p(g), B, GIVEN_LEN, cfg_on)
                lead = bool(g[0, 0] >= 0)
                ends = []
                for n in range(1, n_chain + 1):
                    regs = _regions(lib, h, GIVEN, [B, GIVEN_LEN, cfg_on, n], g)
                    window = ROWS + [INT, INT]
                    _check(regs, size, [INT, INT] + window * n + (ROWS if lead else []), tight=lead)
                    for c in range(n):                   # chain c's window
                        assert (regs[2 + c * 10: 12 + c * 10, 3] == c).all()
                    ends.append(int((regs[:, 0] + regs[:, 1]).max()))
                assert size - max(ends) <= 255
    finally:
        lib.lg_engine_destroy(h)


@pytest.mark.parametrize("conf", [c for c in CONFIGS if c[1] != _lib.LG_DTYPE_F32], ids=_cid)
def test_two_chain_views_split_the_workspace(conf):
    lib = _lib_or_skip()
    h, cfg = _engine(lib, *conf)
    try:
        for rows, seq in [(32, cfg.cls_token_num + 9), (36, 47), (64, cfg.cls_token_num + 16)]:
            full = _regions(lib, h, WS, [rows, seq])
            half = _regions(lib, h, WS, [rows // 2, seq])      # what one chain of rows / 2 rows needs
            views = [_regions(lib, h, WS, [rows, seq, g, 2]) for g in range(2)]
            for g, v in enumerate(views):
                assert v.shape == full.shape and (v[:, 2] == full[:, 2]).all() and (v[:, 3] == g).all()
                for i in range(len(full)):
                    if i in (2 + PARTIAL, len(full) - 1):
                        continue
                    assert full[i, 1] % 2 == 0
                    assert v[i, 1] == full[i, 1] // 2 and v[i, 0] == full[i, 0] + g * v[i, 1], (g, i)
                p, fp = v[2 + PARTIAL], full[2 + PARTIAL]
                assert p[0] % 256 == 0 and p[1] % 256 == 0 and fp[0] <= p[0] and p[0] + p[1] <= full[3 + PARTIAL, 0]   # up to the logits
                assert p[1] >= half[2 + PARTIAL, 1], (p[1], half[2 + PARTIAL, 1])
                c, fc = v[-1], full[-1]
                assert fc[1] == COUNTER_INTS * 4 and c[0] == fc[0] + 8 * g and c[1] == 8
                assert fc[0] <= c[0] + 4 * TICKET and c[0] + 4 * TICKET + 8 <= fc[0] + fc[1]
            p0, p1 = views[0][2 + PARTIAL], views[1][2 + PARTIAL]
            assert p0[0] + p0[1] <= p1[0]
    finally:
        lib.lg_engine_destroy(h)


def test_hook_argument_checks():
    lib = _lib_or_skip()
    h, _ = _engine(lib, _lib.LG_MODEL_C2I, _lib.LG_DTYPE_BF16, 64)
    try:
        out = np.zeros((4, 4), np.int64)
        for kind, args in [(9, [1, 1]), (-1, [1, 1]), (WS, [1]), (WS, [4, 8, 2, 2]), (WS, [3, 8, 0, 2]), (SCORE, [0, 8]),
                           (SJD, [1, 1, 1]), (GIVEN, [1, 4, 1, 1])]:
            a = np.asarray(args, np.int64)
            assert lib.lg_test_scratch_regions(h, kind, _p(a), len(a), None, _p(out), 4) < 0, (kind, args)
        a = np.asarray([2, 8], np.int64)
        assert lib.lg_test_scratch_regions(None, WS, _p(a), 2, None, _p(out), 4) < 0
        n = lib.lg_test_scratch_regions(h, WS, _p(a), 2, None, _p(out), 4)   # more regions than room: the first cap
        assert n == 12 and out[0, 2] == KV and out[1, 0] > out[0, 0]
    finally:
        lib.lg_engine_destroy(h)


@pytest.mark.parametrize("shape", [(12, 768), (16, 1024), (20, 1280), (24, 1536), (32, 2048), (32, 3200)],
                         ids=["GPT-B", "GPT-L", "GPT-XL", "GPT-XXL", "GPT-1B", "GPT-3B"])
def test_registry_shapes_keep_their_partials_region(shape):
    """The workspace's GEMM partials are a whole number of 64-float slices per chain. At the registry's shapes (V = 16384, c2i and t2i,
    CFG batches of 32 to 128 rows) the partials are already a multiple of 128 floats, so that rounding leaves the layout as it was."""
    lib = _lib_or_skip()
    n_head, dim = shape
    for model_type, tc in ((_lib.LG_MODEL_C2I, 1), (_lib.LG_MODEL_T2I, 120)):
        ffn = 256 * ((int(2 * 4 * dim / 3) + 255) // 256)
        cfg = _lib.ModelCfg(2, n_head, dim, ffn, 16384, tc, 256, 1000, 2048, model_type, _lib.LG_DTYPE_BF16, 1e-5)
        h = ctypes.c_void_p()
        assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0, lib.lg_last_error()
        try:
            for rows in (32, 64, 128):
                full = _regions(lib, h, WS, [rows, tc + 256])
                p = full[2 + PARTIAL]
                assert p[1] % (2 * 64 * 4) == 0 and full[3 + PARTIAL, 0] - p[0] == p[1], (rows, p)
        finally:
            lib.lg_engine_destroy(h)
