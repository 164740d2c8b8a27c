"""a10 top-k hard negatives (extension, SURVEY §8 a10): CPU checks of the oracle semantics and of the streamed
radix-select algorithm the kernels implement (contrastiveseg_b200/csrc/pcl_topk.cuh and the top-k modes of
pcl_infonce_simt.cu), emulated step by step in numpy: order-preserving key, 11+11+10-bit levels, warp-lane bin partition,
analytic zero tail, tie weights."""
import numpy as np
import pytest
import torch

from oracle import ref_port as rp

KEY_ZERO = 0x80000000
TK_ALL = 0xFFFFFFFF


def sortable_key(l32: np.ndarray) -> np.ndarray:
    u = l32.astype(np.float32).view(np.uint32).copy()
    u[(u << np.uint32(1)) == 0] = 0                      # -0 -> +0
    neg = (u & np.uint32(0x80000000)) != 0
    return np.where(neg, ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def scan_level(level, hist, prefix, need, tail_count, has_tail):
    """k_topk_scan<LEVEL> for one row.  Returns ('all', total) or ('bin', f_bin, f_rem, f_cnt)."""
    nb = 1024 if level == 3 else 2048
    cb = nb // 32
    tail_bin = -1
    if tail_count > 0 and has_tail:
        if level == 1:
            tail_bin = KEY_ZERO >> 21
        if level == 2 and prefix == (KEY_ZERO >> 21):
            tail_bin = (KEY_ZERO >> 10) & 0x7FF
        if level == 3 and prefix == (KEY_ZERO >> 10):
            tail_bin = KEY_ZERO & 0x3FF
    h = hist[:nb].astype(np.int64).copy()
    if tail_bin >= 0:
        h[tail_bin] += tail_count
    s = np.array([h[nb - (L + 1) * cb: nb - L * cb].sum() for L in range(32)])
    incl = np.cumsum(s)
    above = incl - s
    total = incl[-1]
    mine = (above < need) & (need <= above + s)
    if (level == 1 and total <= need) or not mine.any():
        return ("all", int(total))
    L = int(np.argmax(mine))
    hi, lo = nb - L * cb, nb - (L + 1) * cb
    cum = above[L]
    for b in range(hi - 1, lo - 1, -1):
        if cum + h[b] >= need:
            return ("bin", b, int(need - cum), int(h[b]))
        cum += h[b]
    raise AssertionError("scan did not terminate")


def radix_select_row(keys_neg: np.ndarray, k: int, tail_count: int, has_tail: bool):
    """(tau_key, tie_weight, G, E) of one anchor row exactly as the kernels compute it."""
    hist = np.bincount(keys_neg >> 21, minlength=2048)
    r = scan_level(1, hist, 0, k, tail_count, has_tail)
    if r[0] == "all":
        return 0, 1.0, r[1], 0
    p1, need = r[1], r[2]
    sel = keys_neg[(keys_neg >> 21) == p1]
    hist = np.bincount((sel >> 10) & 0x7FF, minlength=2048)
    r = scan_level(2, hist, p1, need, tail_count, has_tail)
    assert r[0] == "bin"
    p2, need = (p1 << 11) | r[1], r[2]
    sel = keys_neg[(keys_neg >> 10) == p2]
    hist = np.bincount(sel & 0x3FF, minlength=1024)
    r = scan_level(3, hist, p2, need, tail_count, has_tail)
    assert r[0] == "bin"
    tau = (p2 << 10) | r[1]
    return tau, np.float32(r[2]) / np.float32(r[3]), k - r[2], r[3]


def key_to_float(key: int) -> float:
    u = np.uint32(key)
    u = (u & np.uint32(0x7FFFFFFF)) if (u & np.uint32(0x80000000)) else ~u
    return float(np.array([u], dtype=np.uint32).view(np.float32)[0])


def test_sortable_key_is_order_preserving():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.normal(size=2000) * 10, [0.0, -0.0, 1e-30, -1e-30, 3.5, -3.5, 1e30, -1e30]]).astype(np.float32)
    k = sortable_key(x)
    order = np.argsort(x, kind="stable")
    assert np.all(np.diff(k[order].astype(np.int64)) >= 0)
    assert sortable_key(np.array([0.0], np.float32))[0] == KEY_ZERO == sortable_key(np.array([-0.0], np.float32))[0]
    for v in (0.0, 1.0, -2.5, 123.456):
        assert key_to_float(int(sortable_key(np.array([v], np.float32))[0])) == np.float32(v)


@pytest.mark.parametrize("seed,k,tail", [(0, 7, 0), (1, 1, 0), (2, 50, 0), (3, 16, 12), (4, 5, 40), (5, 400, 0), (6, 33, 7)])
def test_radix_select_matches_sort(seed, k, tail):
    """Dyadic data (exact in fp32 and fp64, many ties): the streamed select equals the sort-based oracle weights."""
    g = torch.Generator().manual_seed(seed)
    A, N, D, ncls = 24, 300, 16, 4
    anchors = torch.randint(-3, 4, (A, D), generator=g).double() / 4
    contrast = torch.randint(-3, 4, (N, D), generator=g).double() / 4
    contrast[::7] = 0                                   # exact-zero rows: ties with the analytic tail
    ya = torch.randint(0, ncls, (A,), generator=g)
    yc = torch.randint(1, ncls, (N,), generator=g)
    T = 0.125
    if tail:                                            # bank layout: R zero rows of label 0 appended (Q3)
        contrast_full = torch.cat([contrast, torch.zeros(tail, D, dtype=torch.float64)])
        yc_full = torch.cat([yc, torch.zeros(tail, dtype=torch.long)])
    else:
        contrast_full, yc_full = contrast, yc
    l_full = (anchors @ contrast_full.t()) / T
    same = ya.view(-1, 1) == yc_full.view(1, -1)
    w, tau, G, E = rp.topk_negative_weights(l_full, ~same, k)
    l32 = ((anchors @ contrast.t()) / T).numpy().astype(np.float32)       # streamed columns only
    assert np.array_equal(l32.astype(np.float64), ((anchors @ contrast.t()) / T).numpy())    # exact data
    keys = sortable_key(l32.reshape(-1)).reshape(A, N)
    neg_stream = (ya.view(-1, 1) != yc.view(1, -1)).numpy()
    for i in range(A):
        has_tail = tail > 0 and int(ya[i]) != 0
        tau_key, tw, Gd, Ed = radix_select_row(keys[i][neg_stream[i]], k, tail, has_tail)
        # device weights of the streamed columns + the tail weight
        wd = np.where(keys[i] > tau_key, 1.0, np.where(keys[i] == tau_key, tw, 0.0)) * neg_stream[i]
        assert np.allclose(wd, w[i, :N].numpy(), atol=1e-7), (i, tau_key)
        if has_tail:
            wt = 1.0 if KEY_ZERO > tau_key else (tw if KEY_ZERO == tau_key else 0.0)
            assert np.allclose(wt, w[i, N:].numpy(), atol=1e-7)
        if tau_key != 0:
            assert key_to_float(tau_key) == float(tau[i]) and Gd == int(G[i]) and Ed == int(E[i])
            assert abs(float(wd.sum()) + (tail * wt if has_tail else 0.0) - k) < 1e-4      # exactly k slots
        else:
            assert int(E[i]) == 0 and Gd == int((~same[i]).sum())


def test_oracle_topk_limits():
    """k=None and k >= #negatives reproduce the reference formulation; the k largest are what is summed."""
    g = torch.Generator().manual_seed(11)
    A, N, D = 32, 200, 16
    a = torch.nn.functional.normalize(torch.randn(A, D, generator=g, dtype=torch.float64), dim=1)
    c = torch.nn.functional.normalize(torch.randn(N, D, generator=g, dtype=torch.float64), dim=1)
    ya = torch.randint(0, 5, (A,), generator=g)
    yc = torch.randint(0, 5, (N,), generator=g)
    ref = rp.infonce_closed_form(a, ya, c, yc, 0.1, 0.07, False)
    for k in (None, N, 10 ** 6):
        r = rp.infonce_topk(a, ya, c, yc, 0.1, 0.07, k, False)
        assert torch.equal(r["loss"], ref["loss"]) and torch.equal(r["dA"], ref["dA"])
    k = 9
    r = rp.infonce_topk(a, ya, c, yc, 0.1, 0.07, k, False)
    l = (a @ c.t()) / 0.1
    e = torch.exp(l - l.max(1, keepdim=True).values)
    same = ya.view(-1, 1) == yc.view(1, -1)
    top = torch.where(~same, e, torch.zeros_like(e)).topk(k, dim=1).values.sum(1)
    assert torch.allclose(r["neg"], top, rtol=1e-12)
    assert float(r["loss"]) < float(ref["loss"])        # fewer negatives -> smaller denominator -> smaller loss
    # the analytic gradient equals autograd with the weights held constant
    a2 = a.clone().requires_grad_(True)
    l2 = (a2 @ c.t()) / 0.1
    m = l2.max(1, keepdim=True).values.detach()
    e2 = torch.exp(l2 - m)
    neg = (e2 * r["w"]).sum(1, keepdim=True)
    pos = same.clone()
    pos[torch.arange(A), torch.arange(A)] = False
    loss = (-(0.1 / 0.07) * (((l2 - m) - torch.log(e2 + neg)) * pos).sum(1) / pos.sum(1)).mean()
    loss.backward()
    assert torch.allclose(a2.grad, r["dA"], atol=1e-12)
