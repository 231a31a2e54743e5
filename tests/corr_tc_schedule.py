"""A Python model of the tensor-core correlation's persistent work assignment (correlation_tc.cu), and the batch
shapes that drive it into each of its regimes.  Test helper only.

Both kernels run one CTA per SM over the tiles of the 4 parity classes: a tile is 8 x 16 class pixels (16 x 32 pixels
of the full-resolution image), so a sample of H x W has 4 * ceil(W / 32) * ceil(H / 16) tiles, and a forward tile is
7 units of 4 halo rows.

- Forward (`corr_fwd_tc_kernel`): grid = min(ntiles, sms).  The `full` tiles of whole rounds go round-robin; the
  (tile, unit) pairs of the last, partial round are dealt out in shares of `wper` consecutive pairs, so one CTA's
  share may start inside a tile (ua > 0) and run into the next tile (`tc_next_seg`: one segment per tile).
- Backward (`corr_bwd_tc_kernel`): round-robin over the global tiles [t_begin, t_end) of [0, 2 ntiles); with both
  gradients the even global tiles are gradInput1 tiles and the odd ones the gradInput2 tile of the same location.
"""
TH, TW, NU, UR, DS, DR = 8, 16, 7, 4, 21, 10


def tile_grid(H, W):
    """(nxt, nyt): tiles per class row and column of an H x W image."""
    Hc, Wc = H // 2, W // 2
    return (Wc + TW - 1) // TW, (Hc + TH - 1) // TH


def ntiles(B, H, W):
    nxt, nyt = tile_grid(H, W)
    return 4 * B * nxt * nyt


def decode(t, nxt, nyt):
    """tc_decode: tile index -> (n, py, px, yc0, xc0)."""
    px, q = t & 1, t >> 1
    xc0 = (q % nxt) * TW
    q //= nxt
    yc0 = (q % nyt) * TH
    q //= nyt
    return q >> 1, q & 1, px, yc0, xc0


def tile_of(n, y, x, nxt, nyt):
    """The tile holding full-resolution pixel (y, x) of sample n, and the pixel's row inside the tile."""
    py, px, yc, xc = y & 1, x & 1, y >> 1, x >> 1
    t = ((((n * 2 + py) * nyt + yc // TH) * nxt + xc // TW) << 1) | px
    return t, yc % TH


class Forward(object):
    """corr_fwd_tc_kernel's assignment: `segs[cta]` lists the (tile, ua, ub) segments of each CTA in order, and
    `owner[(tile, unit)]` = (cta, index of the segment in that CTA's list)."""

    def __init__(self, nt, sms):
        self.nt, self.sms, self.grid = nt, sms, min(nt, sms)
        g = self.grid
        self.full = (nt // g) * g
        self.wtotal = (nt - self.full) * NU
        self.wper = (self.wtotal + g - 1) // g
        self.segs, self.owner = [], {}
        for cta in range(g):
            w0 = min(cta * self.wper, self.wtotal)
            w1 = min(w0 + self.wper, self.wtotal)
            tn, w, segs = cta, w0, []
            while True:                                   # tc_next_seg
                if tn < self.full:
                    segs.append((tn, 0, NU))
                    tn += g
                elif w < w1:
                    t, ua = self.full + w // NU, w % NU
                    ub = NU if NU - ua < w1 - w else ua + (w1 - w)
                    w += ub - ua
                    segs.append((t, ua, ub))
                else:
                    break
            for i, (t, ua, ub) in enumerate(segs):
                for u in range(ua, ub):
                    assert (t, u) not in self.owner, "unit (%d, %d) dealt twice" % (t, u)
                    self.owner[(t, u)] = (cta, i)
            self.segs.append(segs)

    def partial_segments(self):
        return [(cta, i, s) for cta, segs in enumerate(self.segs) for i, s in enumerate(segs) if s[0] >= self.full]

    def tiles_per_cta(self):
        return max(len({s[0] for s in segs}) for segs in self.segs)


class Backward(object):
    """corr_bwd_tc_kernel's assignment: `owner[(grad, tile)]` = (cta, how many tiles that CTA ran before it), grad 0 =
    gradInput1, 1 = gradInput2."""

    def __init__(self, nt, sms, need1=True, need2=True):
        t_begin, t_end = (0 if need1 else nt), (2 * nt if need2 else nt)
        both = t_begin == 0 and t_end == 2 * nt
        self.grid = min(t_end - t_begin, sms)
        self.owner, self.per_cta = {}, [0] * self.grid
        for cta in range(self.grid):
            for g in range(t_begin + cta, t_end, self.grid):
                second = (g & 1) if both else int(g >= nt)
                tile = (g >> 1) if both else (g - nt if second else g)
                assert (second, tile) not in self.owner
                self.owner[(second, tile)] = (cta, self.per_cta[cta])
                self.per_cta[cta] += 1

    def tiles_per_cta(self):
        return max(self.per_cta)


# ------------------------------------------------------------------------------------------------
# Regimes, and the shapes that reach them
# ------------------------------------------------------------------------------------------------
def _crosses(f):
    """Some CTA's share of the partial round spans two tiles."""
    return any(len([s for s in segs if s[0] >= f.full]) > 1 for segs in f.segs)


def _starts_inside(f):
    return any(s[1] > 0 for _, _, s in f.partial_segments())


# name -> (what it means, predicate on the forward model of a batch).  Each is reached by the smallest batch of
# 16 x 32 images (4 tiles a sample) that satisfies it, except the ragged ones, which have fixed shapes.
REGIMES = {
    "few": ("fewer tiles than SMs", lambda f: f.nt < f.sms),
    "rounds": ("whole rounds, no partial round", lambda f: f.nt >= f.sms and f.wtotal == 0),
    "wper1": ("a partial round of one unit per CTA", lambda f: f.full > 0 and f.wper == 1),
    "wper2": ("shares of 2 units, some spanning two tiles", lambda f: f.full > 0 and f.wper == 2 and _crosses(f)),
    "wper5": ("shares of 5 units", lambda f: f.full > 0 and f.wper == 5),
    "wper6": ("shares of 6 units, segments starting at ua > 0",
              lambda f: f.full > 0 and f.wper == 6 and _starts_inside(f)),
    "rounds3": ("3 full rounds and a partial one", lambda f: f.full == 3 * f.grid and f.wtotal > 0),
    "ragged4": ("samples of 9 tiles a class, ragged in both dims", lambda f: True),
    "ragged11": ("samples of 9 tiles a class, ragged in both dims", lambda f: True),
}
RAGGED = {"ragged4": (4, 34, 70), "ragged11": (11, 34, 70)}


def pick(regime, sms, max_batch=1024):
    """(B, H, W) of the batch that reaches `regime` on a GPU with `sms` SMs."""
    if regime in RAGGED:
        return RAGGED[regime]
    pred = REGIMES[regime][1]
    for B in range(1, max_batch + 1):
        if pred(Forward(ntiles(B, 16, 32), sms)):
            return B, 16, 32
    raise ValueError("no batch of 16 x 32 images up to %d reaches %s at %d SMs" % (max_batch, regime, sms))


def describe(B, H, W, sms):
    f = Forward(ntiles(B, H, W), sms)
    b = Backward(f.nt, sms)
    return "B%d-%dx%d-t%d-full%d-wper%d-fwd%d-bwd%d" % (B, H, W, f.nt, f.full, f.wper, f.tiles_per_cta(), b.tiles_per_cta())


def locate_forward(f, H, W, n, d, y, x):
    """Where output element (n, d, y, x) was computed: 'sample n class (py,px) tile t unit u CTA c segment i'."""
    nxt, nyt = tile_grid(H, W)
    t, row = tile_of(n, y, x, nxt, nyt)
    u = (d // DS + row) // UR
    cta, i = f.owner[(t, u)]
    ua, ub = f.segs[cta][i][1:]
    part = "partial round" if t >= f.full else "round %d" % (t // f.grid)
    return "sample %d class (%d,%d) tile %d unit %d CTA %d segment %d [units %d..%d, %s]" % (
        n, y & 1, x & 1, t, u, cta, i, ua, ub - 1, part)


def locate_backward(b, H, W, grad, n, y, x):
    nxt, nyt = tile_grid(H, W)
    t, row = tile_of(n, y, x, nxt, nyt)
    cta, k = b.owner[(grad, t)]
    return "gradInput%d sample %d class (%d,%d) tile %d warpgroup %d CTA %d (its tile #%d)" % (
        grad + 1, n, y & 1, x & 1, t, row // 4, cta, k)
