"""A vectorised numpy restatement of match::stereo::compute (OpenVSLAM match/stereo.cc; ORB-SLAM2's ComputeStereoMatches
apart from the median factor, DESIGN.md section 5), written from the reference's semantics, not from the oracle or the kernel.

For every left keypoint:

* rows: the keypoint's row is int(y_left) (truncation) and must lie in [0, rows of level 0); a right keypoint of octave o
  covers the rows [floor(y - 2 s[o]), ceil(y + 2 s[o])], the bounds formed in float32;
* candidates: |o_r - o_l| <= 1 and x_left - max_disp <= x_right <= x_left - 0 (float32, inclusive), max_disp =
  float32(focal_x_baseline / true_baseline); the nearest descriptor wins, the lowest right index on ties, and it must be
  closer than (HAMMING_DIST_THR_HIGH + HAMMING_DIST_THR_LOW) / 2 = 75;
* SAD: on the left octave's pyramid level, sxl, syl, sxr = rint(float32(x * inv_s)) (round half to even); the right
  windows of the 11 offsets and the left window must lie inside the level; each 11 x 11 window minus its centre pixel;
  the first minimum over the offsets -5..5 wins, and a minimum at -5 or 5 is rejected;
* sub-pixel: delta = float32(float32(c1 - c3) / (2 (float32(c1 + c3) - 2 c2))), the division and the outer sums in
  float64; x_right = float32(s * float32(float32(sxr + off) + delta)), disp = float32(x_left - x_right);
* disparity: disp < 0 or disp >= max_disp is rejected; disp == 0 becomes 0.01 (x_right = x_left - 0.01);
  depth = float32(focal_x_baseline / disp);
* median test: the accepted (SAD, left index) pairs sorted; from the largest down, a match is dropped while its SAD is
  at least 2 x the SAD at index size // 2.  The count returned is the number of matches before this test.

A keypoint with a coordinate that is not finite takes no part: a left one is not matched, a right one is no candidate.
The reference leaves these undefined (its float to int conversions); the kernel and the oracle gate them explicitly.

The bound on delta: the minimum at the best offset is strict on the left (first minimum) and weak on the right, so
c1 > c2 and c3 >= c2.  Then c1 + c3 - 2 c2 >= c1 - c2 > 0 and |c1 - c3| <= c1 + c3 - 2 c2 with c1 - c3 = c1 + c3 - 2 c2
only when c3 == c2, so delta lies in (-0.5, 0.5].  The reference's |delta| > 1 rejection (kept in the kernel and the
oracle) can never fire; compute() asserts the bound on every match.

numpy's float32 arithmetic rounds to nearest like the kernel's __f*_rn and the oracle's -ffp-contract=off C, so
x_right and depth are bit-exact.  compute() also evaluates x_right and depth in float64 from the same integer SADs."""
import numpy as np

HAMMING_THR = (100 + 50) // 2
WIN, SLIDE = 5, 5

REASONS = ("not_finite", "row_outside", "max_x_right_negative", "no_candidate_below_threshold", "right_window_outside",
           "left_window_outside", "best_offset_at_edge", "disparity_out_of_range", "clamped_zero_disparity",
           "median_rejected", "matched")
R = {name: k for k, name in enumerate(REASONS)}

f32 = np.float32


def _words(desc):
    return np.ascontiguousarray(desc, np.uint8).reshape(-1, 32).view(np.uint64)


def _best_candidates(row, lx, lo, ld, rx, ry, ro, rd, sf, max_disp, live):
    """-> (best right index or -1, best distance) of each left keypoint: the first nearest candidate below the threshold."""
    nl, nr = len(lx), len(rx)
    best = np.full(nl, -1, np.int64)
    bestd = np.full(nl, 256, np.int64)
    if nr == 0 or not live.any():
        return best, bestd
    r = (f32(2.0) * sf[ro]).astype(f32)
    with np.errstate(invalid="ignore", over="ignore"):
        lo_row = np.floor((ry - r).astype(f32)).astype(np.float64)
        hi_row = np.ceil((ry + r).astype(f32)).astype(np.float64)
    rfin = np.isfinite(rx) & np.isfinite(ry)
    min_xr = (lx - f32(max_disp)).astype(f32)
    max_xr = (lx - f32(0.0)).astype(f32)
    lw, rw = _words(ld), _words(rd)
    todo = np.flatnonzero(live)
    chunk = max(1, (1 << 21) // nr)
    for c0 in range(0, len(todo), chunk):
        idx = todo[c0:c0 + chunk]
        cand = rfin[None, :] & (lo_row[None, :] <= row[idx, None]) & (row[idx, None] <= hi_row[None, :])
        cand &= np.abs(ro[None, :].astype(np.int64) - lo[idx, None]) <= 1
        cand &= (min_xr[idx, None] <= rx[None, :]) & (rx[None, :] <= max_xr[idx, None])
        d = np.bitwise_count(lw[idx][:, None, :] ^ rw[None, :, :]).sum(-1, dtype=np.int64)
        d = np.where(cand, d, 256)
        j = np.argmin(d, axis=1)                       # argmin returns the first index of the minimum
        dj = d[np.arange(len(idx)), j]
        ok = dj < HAMMING_THR
        best[idx[ok]] = j[ok]; bestd[idx[ok]] = dj[ok]
    return best, bestd


def compute(left_pyr, right_pyr, scale_factors, kps_left, desc_left, kps_right, desc_right, focal_x_baseline, true_baseline):
    """-> dict(x_right, depth (float32, -1 where unmatched), num_matched (before the median test), reason (index into
    REASONS per left keypoint), sad (int64, -1 where no SAD was taken), best_right (-1 without a candidate),
    x_right64 / depth64 (float64 from the same SADs, NaN where unmatched))."""
    sf = np.asarray(scale_factors, f32)
    inv_sf = (f32(1.0) / sf).astype(f32)
    lx = np.asarray(kps_left["x"], f32); ly = np.asarray(kps_left["y"], f32); lo = np.asarray(kps_left["octave"], np.int64)
    rx = np.asarray(kps_right["x"], f32); ry = np.asarray(kps_right["y"], f32); ro = np.asarray(kps_right["octave"], np.int64)
    fxb = f32(focal_x_baseline)
    max_disp = f32(fxb / f32(true_baseline))
    nl = len(lx)
    rows0 = left_pyr[0].shape[0]
    reason = np.full(nl, -1, np.int64)
    xr_out = np.full(nl, -1, f32); dp_out = np.full(nl, -1, f32)
    xr64 = np.full(nl, np.nan); dp64 = np.full(nl, np.nan)
    sad_out = np.full(nl, -1, np.int64)

    fin = np.isfinite(lx) & np.isfinite(ly)
    reason[~fin] = R["not_finite"]
    row = np.where(fin, np.trunc(np.where(fin, ly, 0).astype(np.float64)), 0.0)
    row_ok = fin & (0 <= row) & (row < rows0)
    reason[fin & ~row_ok] = R["row_outside"]
    xneg = row_ok & ((lx - f32(0.0)).astype(f32) < 0)
    reason[xneg] = R["max_x_right_negative"]
    live = row_ok & ~xneg

    best, _ = _best_candidates(row, lx, lo, desc_left, rx, ry, ro, desc_right, sf, max_disp, live)
    reason[live & (best < 0)] = R["no_candidate_below_threshold"]

    accepted = []
    for il in np.flatnonzero(live & (best >= 0)):
        lvl = int(lo[il]); ir = int(best[il])
        inv_s = inv_sf[lvl]
        sxl = float(np.rint(f32(lx[il] * inv_s))); syl = float(np.rint(f32(ly[il] * inv_s))); sxr = float(np.rint(f32(rx[ir] * inv_s)))
        Lp, Rp = left_pyr[lvl], right_pyr[lvl]
        H, W = Lp.shape
        if sxr - SLIDE - WIN < 0 or W <= sxr + SLIDE + WIN + 1:
            reason[il] = R["right_window_outside"]; continue
        if sxl - WIN < 0 or W <= sxl + WIN or syl - WIN < 0 or H <= syl + WIN:
            reason[il] = R["left_window_outside"]; continue
        sxl, syl, sxr = int(sxl), int(syl), int(sxr)
        a = Lp[syl - WIN:syl + WIN + 1, sxl - WIN:sxl + WIN + 1].astype(np.int64) - int(Lp[syl, sxl])
        sads = np.empty(2 * SLIDE + 1, np.int64)
        for k, off in enumerate(range(-SLIDE, SLIDE + 1)):
            c = sxr + off
            b = Rp[syl - WIN:syl + WIN + 1, c - WIN:c + WIN + 1].astype(np.int64) - int(Rp[syl, c])
            sads[k] = np.abs(a - b).sum()
        k = int(np.argmin(sads))
        sad_out[il] = sads[k]
        if k == 0 or k == 2 * SLIDE:
            reason[il] = R["best_offset_at_edge"]; continue
        off = k - SLIDE
        c1, c2, c3 = f32(sads[k - 1]), f32(sads[k]), f32(sads[k + 1])
        delta = f32(np.float64(f32(c1 - c3)) / (2.0 * (np.float64(f32(c1 + c3)) - 2.0 * np.float64(c2))))
        assert -0.5 < delta <= 0.5, (il, sads)
        x_right = f32(sf[lvl] * f32(f32(sxr + off) + delta))
        disp = f32(lx[il] - x_right)
        if disp < 0 or max_disp <= disp:
            reason[il] = R["disparity_out_of_range"]; continue
        d64 = (float(sads[k - 1]) - float(sads[k + 1])) / (2.0 * (float(sads[k - 1]) + float(sads[k + 1]) - 2.0 * float(sads[k])))
        x64 = float(sf[lvl]) * (sxr + off + d64)
        if disp == 0:
            disp = f32(0.01); x_right = f32(lx[il] - disp)
            reason[il] = R["clamped_zero_disparity"]
            dp64[il] = float(fxb) / float(disp); xr64[il] = float(lx[il]) - float(disp)
        else:
            reason[il] = R["matched"]
            dp64[il] = float(fxb) / (float(lx[il]) - float(x_right)); xr64[il] = x64
        xr_out[il] = x_right; dp_out[il] = f32(fxb / disp)
        accepted.append((int(sads[k]), int(il)))

    if accepted:
        accepted.sort()
        thr = f32(2.0) * f32(accepted[len(accepted) // 2][0])
        for sad, il in reversed(accepted):
            if f32(sad) < thr:
                break
            xr_out[il] = -1; dp_out[il] = -1; xr64[il] = np.nan; dp64[il] = np.nan
            reason[il] = R["median_rejected"]
    assert (reason >= 0).all()
    return dict(x_right=xr_out, depth=dp_out, num_matched=len(accepted), reason=reason, sad=sad_out, best_right=best,
                x_right64=xr64, depth64=dp64)
