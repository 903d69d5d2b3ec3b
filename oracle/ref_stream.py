"""The pieces every chunked CPU stream reference shares (TEST INFRASTRUCTURE): carrying a history, reading rows of
[history | chunk], a conv over them, driving a reference through a push schedule, and measuring a whole-utterance
model's lookahead by autograd."""
import torch
import torch.nn.functional as F


def keep(x, h, short=0):
    """the last ``h`` samples of x as the history to carry, zero-extended on the left (``short``: that many of the oldest
    lost, zero instead)"""
    if h == 0:
        return x[..., :0]
    kept = x[..., max(x.shape[-1] - h, 0) + short:]
    return F.pad(kept, (h - kept.shape[-1], 0))


def rows(hist, x, first, n):
    """rows [first, first + n) of [hist | x], row 0 being x's first"""
    xp = torch.cat([hist, x], -1)
    H = hist.shape[-1]
    assert 0 <= H + first and H + first + n <= xp.shape[-1], (H, first, n, xp.shape)
    return xp[..., H + first:H + first + n]


def conv(hist, x, w, b, d, slope, pad_left, n):
    """n outputs of the conv of lrelu([hist | x]) whose first output reads row -pad_left"""
    k = w.shape[-1]
    xs = rows(hist, x, -pad_left, n + (k - 1) * d)
    return F.conv1d(F.leaky_relu(xs, slope), w, b, dilation=d)


def drive(push, T, schedule, flush=None, first=None):
    """Push a T-frame utterance in chunks of ``schedule`` frames (after a first chunk of ``first`` frames if given;
    repeated until the utterance is used up, the last chunk cut short), then ``flush()`` if given; returns the outputs
    concatenated.  ``push(j, n)`` pushes frames [j, j + n)."""
    outs, j, k = [], 0, 0
    if first:
        outs.append(push(0, first))
        j = first
    while j < T:
        n = min(schedule[k % len(schedule)], T - j)
        outs.append(push(j, n))
        j, k = j + n, k + 1
    if flush is not None:
        outs.append(flush())
    return torch.cat(outs, -1)


def measured_lookahead(whole, x, frame, hop, rate=1):
    """The true lookahead of a whole-utterance model in output samples, measured by float64 autograd: frame * hop - o for
    the first output sample o of ``whole(x)`` that depends on input frame ``frame`` of x (1, C, frames * rate, requires
    grad; ``rate`` input samples per frame).  The dependency is shift-invariant by a frame, so a binary search over the
    outputs up to that frame's last finds it."""
    y = whole(x)

    def depends(o):
        (gx,) = torch.autograd.grad(y[0, 0, o], x, retain_graph=True)
        return bool(gx[0, :, frame * rate:(frame + 1) * rate].abs().sum() > 0)

    lo, hi = 0, (frame + 1) * hop - 1
    assert depends(hi) and not depends(0)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (lo, mid) if depends(mid) else (mid, hi)
    return frame * hop - hi
