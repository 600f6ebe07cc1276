"""The TargetDiff, DiffBP and DiffSBDD validation-loss stages against float64 at their per-graph edges.

Each loss kernel (eval_loss_kernel, bp_eval_loss_kernel, sbdd_eval_loss_kernel) and the DiffSBDD noise kernel runs one
CTA of 128 threads per (replica, graph): a strided loop over the graph's ligand atoms feeds block_sum, which adds four
warp partials as (w0 + w1) + (w2 + w3).  Every input of a loss stage is returned by the call (the denoiser's outputs) or
rebuilt from its draws, so a float64 restatement of the stage, fed the call's own outputs and the fp32 coefficients the
kernel received (``model.eval_coef(t)``), is checked against it at fp32-rounding bars.

Layouts, each through the production ``eval_losses`` (pocket atoms, ligand atoms) per graph:
- 'sizes': ligands of 1, 31, 32, 33, 127, 128, 129, 256 and 257 atoms (DiffBP, which returns per-timestep but no
  per-graph values, runs each size as a batch of its own: 'lig<n>_alone');
- 'lig1500': ligandless graphs between and after others around a 1500-atom ligand;
- 'partial': partial generation with context atoms spread across thread strides and whole warps, a graph whose ligand
  is all context between generated graphs, and a graph without a pocket;
- 'nothing_generated': every ligand atom is context (TargetDiff and DiffBP losses NaN, DiffBP atom loss 0).
Timesteps: several replicas of distinct t in one call, t in {0, 1, T/2, T - 1} (TargetDiff, DiffBP) and {1, 2, T/2, T}
(DiffSBDD) of a T = 1000 schedule.  Class counts: 13 (the shipped count) and 16 (CBG_MAXCLS) for all three models.
The DiffSBDD model zeroes the last Linear of every ``xv_func``: its coordinate update is then exactly 0, so the t = 0
copy's prediction (which no call returns) is the noised input position and all six per-graph terms are checked; one
case with the seeded ``xv_func`` checks the five terms that do not need it.

Noise stage: TargetDiff x_t against float64 within a few ulps, v_t against the float64 Gumbel-max class on rows whose
top-two margin exceeds its bar (skipped rows counted, at most 1 %); the DiffBP mask exactly, with u equal to the mask
probability and one ulp either side.  Quirks exactly: the scatter-mean row count of the per-t losses (recomputed in fp32
from the per-graph values), DiffBP's atom loss of 0 without masked atoms, DiffSBDD's terms of a graph without ligand
atoms (d = -3).  Determinism: repeated calls and a forced split (``max_nodes``) are bit-identical to one launch.

Bars (per element, float64), derived from the magnitudes of the element's intermediates, never from the result:
ULPS fp32 ulps of every intermediate the kernel rounds, probability-weighted over classes for the type KL; a CDF
difference in the Gaussian tail is bounded by its conditioning (pdf x argument error plus the rounding of the CDFs near
1); the interior loss's 48-neighbour cut adds whole terms to the bar only where the 49th distance lies within the bars
of the 48th; a per-graph sum adds (ceil(n_g / 128) + 8) * 2^-24 * sum |z| (the depth of the fixed-order sum), a per-replica mean
over B rows (B + 3) * 2^-24 * mean |z|.  Each check reports how many elements it holds to a tight bar (within 1e-5 of
the result or, where the result cancels, of its largest intermediate) and requires a minimum share of them, so that
loose bars cannot hollow the test out."""
import math

import numpy as np
import pytest
import torch
from scipy.special import erfc

from cbgbench_b200 import synthetic
from cbgbench_b200.diffbp import DiffBPB200
from cbgbench_b200.diffsbdd import DiffSBDDB200
from helpers import make_model, to_dev

torch.set_grad_enabled(False)
T_SCHED = 1000
T_TD = (0, 1, T_SCHED // 2, T_SCHED - 1)
T_SBDD = (1, 2, T_SCHED // 2, T_SCHED)
KS = (13, 16)
ULPS = 6
U32 = 2.0 ** -24
LOG1E30 = float(np.int32(-1031133259).view(np.float32))     # fp32 log(1e-30), the kernels' log_1e30()
SQRT1_2 = math.sqrt(0.5)

SIZES = (1, 31, 32, 33, 127, 128, 129, 256, 257)
# (pocket atoms, ligand atoms) per graph, and per graph which ligand atoms are generated
LAYOUTS = {
    'sizes': ([(24, n) for n in SIZES], 'all'),
    'lig1500': ([(30, 20), (25, 0), (300, 1500), (12, 0)], 'all'),
    'partial': ([(40, 300), (30, 150), (0, 260), (20, 129)], ['strided', 'none', 'strided', 'strided']),
    'nothing_generated': ([(30, 20), (20, 140)], ['none', 'none']),
}
# DiffBP returns no per-graph values: its size edges run one graph per batch, so that no graph's error is diluted
SINGLES = {f'lig{n}_alone': ([(24, n)], 'all') for n in SIZES}
BP_LAYOUTS = list(SINGLES) + ['lig1500', 'partial', 'nothing_generated']


def _strided(n):
    """Context atoms at two residues mod 7 and in every fourth warp-sized run: spread over thread strides and warps."""
    a = np.arange(n)
    return ~((a % 7 == 0) | (a % 7 == 3) | ((a // 32) % 4 == 1))


def _batch(layout, K, seed):
    graphs, gen_mode = {**LAYOUTS, **SINGLES}[layout]
    batch = synthetic.make_batch([p for p, _ in graphs], [n for _, n in graphs], seed=seed, num_classes=K)
    modes = [gen_mode] * len(graphs) if isinstance(gen_mode, str) else gen_mode
    gen = [{'all': np.ones(n, bool), 'none': np.zeros(n, bool), 'strided': _strided(n)}[m] for (_, n), m in zip(graphs, modes)]
    batch['ligand_gen_flag'] = torch.from_numpy(np.concatenate(gen))
    return batch


def _sp(a):
    """fp32 ulp of |a| (float64 in, float64 out); 0 for an exact 0, which fp32 holds without rounding."""
    a = np.abs(np.asarray(a, np.float64))
    return np.where(a == 0, 0.0, np.spacing(a.astype(np.float32)).astype(np.float64))


def _np(t):
    return t.detach().cpu().double().numpy() if torch.is_tensor(t) else np.asarray(t, np.float64)


class Checks:
    """Element-wise |got - want| <= bar with NaN == NaN, and a count of the elements held to a tight bar."""

    def __init__(self, tag):
        self.tag, self.lines = tag, []

    def __call__(self, what, got, want, bar, min_tight=0.5, scale=0.0):
        """``scale``: the magnitude of the element's largest intermediate where the result cancels below it; an
        element is tight when its bar is within 1e-5 of max(|want|, scale)."""
        scale = np.broadcast_to(np.asarray(scale, np.float64), np.shape(want)).ravel()
        got, want, bar = (np.broadcast_to(np.asarray(v, np.float64), np.shape(want)).ravel() for v in (got, want, bar))
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan), f'{self.tag} {what}: NaN pattern differs'
        g, w, b, sc = got[~nan], want[~nan], bar[~nan], scale[~nan]
        assert np.all(np.isfinite(b)), f'{self.tag} {what}: non-finite bar'
        bad = np.abs(g - w) > b
        if bad.any():
            i = int(np.argmax(np.abs(g - w) - b))
            raise AssertionError(f'{self.tag} {what}: {int(bad.sum())} of {w.size} elements outside their bars; worst got '
                                 f'{g[i]:.9g} want {w[i]:.9g} bar {b[i]:.3g}')
        tight = int((b <= 1e-5 * np.maximum(np.abs(w), sc)).sum())
        self.lines.append(f'{what} {tight}/{w.size} tight')
        assert w.size == 0 or tight >= min_tight * w.size, f'{self.tag} {what}: only {tight} of {w.size} bars tight'

    def report(self):
        print(f'[{self.tag}] ' + '; '.join(self.lines))


def _graph_mean(e, bar, sel, bl, n_all, B):
    """Per-graph mean of e over the selected atoms (0 without any), its bar, and the selected counts."""
    cnt = np.bincount(bl[sel], minlength=B).astype(np.float64)
    c1 = np.maximum(cnt, 1)
    s = np.bincount(bl[sel], e[sel], minlength=B)
    sa = np.bincount(bl[sel], np.abs(e[sel]), minlength=B)
    sb = np.bincount(bl[sel], bar[sel], minlength=B)
    depth = np.ceil(n_all / 128) + 8
    m = s / c1
    return m, np.where(cnt > 0, (sb + depth * U32 * sa) / c1 + _sp(m), 0.0), cnt      # 0 / 1 is exact


def _rows_mean(m, bar, last):
    """The per-replica mean over graph rows 0 .. last (NaN without rows) and its bar."""
    if last < 0:
        return math.nan, 0.0
    v = m[:last + 1]
    return float(v.mean()), float(bar[:last + 1].mean() + (last + 4) * U32 * np.abs(v).mean())


def _fp32_rows_mean(gl, last):
    """The reduce kernels' fp32 sequential sum over rows 0 .. last, divided by last + 1."""
    if last < 0:
        return np.float32(np.nan)
    s = np.float32(0)
    for v in np.asarray(gl, np.float32)[:last + 1]:
        s = np.float32(s + v)
    return np.float32(s / np.float32(last + 1))


def _common(batch):
    bl = batch['ligand_element_batch'].numpy()
    B = int(torch.cat([batch['ligand_element_batch'], batch['protein_element_batch']]).max()) + 1
    n_all = np.bincount(bl, minlength=B).astype(np.float64)
    return bl, B, n_all, batch['ligand_gen_flag'].numpy()


_MODELS = {}


def _model(kind, K):
    key = (kind, K)
    if key not in _MODELS:
        if kind == 'td':
            m = make_model(T_SCHED, 'cuda', num_layers=1, num_atomtype=K)[0]
        else:
            cls, cfg = {'bp': (DiffBPB200, synthetic.diffbp_config(num_steps=T_SCHED, num_layers=1, num_atomtype=K,
                                                                    num_layers_com=1)),
                        'sbdd': (DiffSBDDB200, synthetic.diffsbdd_config(num_steps=T_SCHED, num_layers=1, num_atomtype=K)),
                        'sbdd_xv': (DiffSBDDB200, synthetic.diffsbdd_config(num_steps=T_SCHED, num_layers=1,
                                                                            num_atomtype=K))}[kind]
            m = cls(cfg)
            sd = synthetic.seeded_state_dict(m, seed=0)
            if kind == 'sbdd':                   # no coordinate update: the prediction of a copy is its input position
                sd = {k: torch.zeros_like(v) if 'xv_func.net.3' in k else v for k, v in sd.items()}
            m.load_state_dict(sd, strict=True)
            m = m.eval().to('cuda')
        _MODELS[key] = m
    return _MODELS[key]


# ---- TargetDiff -------------------------------------------------------------------------------------------------------

def _q_v_posterior(lv0, vt, cf, K):
    """q_v_posterior in float64 -> (log posterior, A, B, lse) [n, K]."""
    logK = math.log(K)
    hot = np.arange(K)[None] == vt[:, None]
    A = np.logaddexp(lv0 + cf.log_alphas_cumprod_prev, cf.log_one_minus_alphas_cumprod_prev - logK)
    Bm = np.logaddexp(np.where(hot, 0.0, LOG1E30) + cf.log_alpha, cf.log_one_minus_alpha - logK)
    o = A + Bm
    mx = o.max(1, keepdims=True)
    lse = mx + np.log(np.exp(o - mx).sum(1, keepdims=True))
    return o - lse, A, Bm, lse


def _td_check(model, batch, t_values, seed, ck):
    K = model.num_classes
    bl, B, n_all, gen = _common(batch)
    n, R = bl.shape[0], len(t_values)
    pn, tu = synthetic.make_noise(R, n, K, seed=seed)
    loss, res = model.eval_losses(to_dev(batch), t_values, pos_noise=pn, type_uniform=tu)
    gl = _np(model.last_graph_loss)
    assert gl.shape == (R, B, 2)
    x0, v0 = _np(batch['ligand_pos']), batch['ligand_atom_type'].numpy()
    hot0 = np.arange(K)[None] == v0[:, None]
    lc0 = np.where(hot0, 0.0, LOG1E30)
    reps, rep_bars, per_t32 = [], [], []
    skipped = gen_rows = 0
    for r, t in enumerate(t_values):
        cf = model.eval_coef(t)
        eps, u = _np(pn[r]), _np(tu[r])
        # noise stage: x_t, and v_t = argmax(log q(v_t | v_0) + Gumbel(u))
        sa, s1 = math.sqrt(cf.alphas_cumprod), math.sqrt(1.0 - cf.alphas_cumprod)
        g3 = gen[:, None]
        ck('xt', _np(res[r]['xt']), np.where(g3, sa * x0 + s1 * eps, x0),
           np.where(g3, ULPS * (_sp(sa * x0) + _sp(s1 * eps)), 0.0), min_tight=0.9)
        vt = res[r]['vt'].cpu().numpy()
        lq = np.logaddexp(lc0 + cf.log_alphas_cumprod, cf.log_one_minus_alphas_cumprod - math.log(K))
        gum = -np.log(-np.log(u + 1e-30) + 1e-30)
        score = gum + lq
        top = np.sort(score, 1)
        margin = top[:, -1] - top[:, -2]
        mbar = 2 * ULPS * (_sp(np.abs(lq).max(1)) + _sp(np.abs(gum).max(1)) + 4 * U32)
        ok = gen & (margin > mbar)
        assert np.array_equal(vt[ok], score.argmax(1)[ok]), f't={t}: v_t differs from the float64 Gumbel-max class'
        assert np.array_equal(vt[~gen], v0[~gen]), f't={t}: a context atom changed type'
        skipped += int((gen & ~ok).sum())
        gen_rows += int(gen.sum())
        # loss stage from the call's own x_pred, c_pred and v_t
        d = _np(res[r]['x_pred']) - x0
        pos_e = (d * d).sum(1)
        pos_b = ULPS * _sp(pos_e)
        with np.errstate(divide='ignore'):
            lcp = np.log(_np(res[r]['c_pred']))
        lpt, At, Bt, lt = _q_v_posterior(lc0, vt, cf, K)
        lpp, Ap, Bp, lp = _q_v_posterior(lcp, vt, cf, K)
        e_c = ULPS * (_sp(At) + _sp(Bt) + _sp(Ap) + _sp(Bp) + _sp(lt) + _sp(lp)
                      + _sp(np.where(np.isfinite(lcp), lcp, 0.0)) + 4 * U32)
        p = np.exp(lpt)
        kl_terms = p * (lpt - lpp)
        kl = kl_terms.sum(1)
        kl_b = (p * e_c * (2 + np.abs(lpt - lpp))).sum(1) + K * U32 * np.abs(kl_terms).sum(1) + _sp(kl)
        nll = -(np.exp(lc0) * lpp).sum(1)
        nll_b = e_c[hot0] + K * U32 * np.abs(nll) + _sp(nll)
        atom_e, atom_b = (nll, nll_b) if t == 0 else (kl, kl_b)
        pm, pb, cnt = _graph_mean(pos_e, pos_b, gen, bl, n_all, B)
        am, ab, _ = _graph_mean(atom_e, atom_b, gen, bl, n_all, B)
        ck('graph pos', gl[r, :, 0], pm, pb, min_tight=0.9)
        ck('graph atom', gl[r, :, 1], am, ab, scale=-LOG1E30)     # cancels from terms of size |log 1e-30|
        last = int(np.nonzero(cnt)[0].max()) if cnt.any() else -1
        reps.append([_rows_mean(pm, pb, last)[0], _rows_mean(am, ab, last)[0]])
        rep_bars.append([_rows_mean(pm, pb, last)[1], _rows_mean(am, ab, last)[1]])
        # scatter_mean row count: trailing graphs dropped, zero-count rows inside the range counted as 0, exactly
        assert np.all(gl[r, cnt == 0] == 0.0)
        per_t32.append([_fp32_rows_mean(gl[r, :, k], last) for k in (0, 1)])
    reps, rep_bars = np.array(reps), np.array(rep_bars)
    for i, k in enumerate(('pos', 'atom')):
        assert torch.equal(loss[k], torch.mean(torch.tensor([float(v[i]) for v in per_t32]))) or \
            (math.isnan(float(loss[k])) and math.isnan(float(per_t32[0][i]))), f'{k}: per-t reduction differs'
        ck(f'loss {k}', float(loss[k]), reps[:, i].mean(), rep_bars[:, i].mean() + (R + 3) * U32 * np.abs(reps[:, i]).mean(),
           scale=-LOG1E30 if k == 'atom' else 0.0)
    assert skipped <= 0.01 * max(gen_rows, 1), f'{skipped} of {gen_rows} v_t rows within their margin bar'
    ck.lines.append(f'v_t {gen_rows - skipped}/{gen_rows} rows checked')
    return loss


@pytest.mark.gpu
@pytest.mark.parametrize('K', KS)
@pytest.mark.parametrize('layout', list(LAYOUTS))
def test_targetdiff_loss_against_float64(layout, K):
    ck = Checks(f'targetdiff {layout} K={K}')
    loss = _td_check(_model('td', K), _batch(layout, K, seed=11), T_TD, seed=12, ck=ck)
    if layout == 'nothing_generated':
        assert math.isnan(float(loss['pos'])) and math.isnan(float(loss['atom']))
    ck.report()


# ---- DiffBP -----------------------------------------------------------------------------------------------------------

def _crafted_u(tu, model, t_values):
    """type_uniform with u equal to the mask probability and one ulp either side on atoms 0, 1, 2 mod 5."""
    tu = tu.clone()
    n = tu.shape[1]
    for r, t in enumerate(t_values):
        mp = np.float32(model.eval_coef(t).mask_prob)
        vals = [mp, np.nextafter(mp, np.float32(2)), np.nextafter(mp, np.float32(-1)) if mp > 0 else mp]
        for k, v in enumerate(vals):
            tu[r, k::5] = float(v)
    return tu


def _bp_inter(xs, xs_b, prot, bl, bp, B):
    """Interior loss terms per ligand atom in float64, with bars: for each protein atom its min(48, n_g) nearest ligand
    atoms of the graph (ties to the lower index).  Where the 49th distance lies within the bars of the 48th the cut
    itself is uncertain: then every pair within its bar of the cut adds its whole term to the bar.  Also returns the
    magnitude 5 + |lpl| of each atom's largest intermediate (0 where the hinge clips exactly)."""
    out, bar, mag = np.zeros(xs.shape[0]), np.zeros(xs.shape[0]), np.zeros(xs.shape[0])
    for g in range(B):
        li, pi = np.nonzero(bl == g)[0], np.nonzero(bp == g)[0]
        if li.size == 0:
            continue
        L, P, Lb = xs[li], prot[pi], xs_b[li]
        diff = P[:, None, :] - L[None, :, :]
        d2 = (diff * diff).sum(-1)                                                  # [np, nl]
        d2b = ULPS * _sp(d2) + 2 * (np.abs(diff) * Lb[None]).sum(-1)
        sel = np.ones_like(d2, bool)
        amb = np.zeros_like(d2, bool)
        if li.size > 48:
            order = np.lexsort((np.broadcast_to(np.arange(li.size), d2.shape), d2), axis=1)
            rank = np.empty_like(order)
            np.put_along_axis(rank, order, np.arange(li.size)[None].repeat(d2.shape[0], 0), axis=1)
            sel = rank < 48
            kth = np.take_along_axis(d2, order[:, 47:48], 1)
            kb = np.take_along_axis(d2b, order[:, 47:48], 1)
            nxt = np.take_along_axis(d2, order[:, 48:49], 1)
            nb = np.take_along_axis(d2b, order[:, 48:49], 1)
            amb = (nxt - kth <= nb + kb) & (np.abs(d2 - kth) <= d2b + kb)
        term = np.exp(-0.5 * d2)
        s = (sel * term).sum(0)
        sb = (sel * term * (0.5 * d2b + ULPS * U32)).sum(0) + (amb * term).sum(0) + P.shape[0] * U32 * s
        lpl = -2 * np.log(s + 1e-3)
        lb = 2 * sb / (s + 1e-3) + ULPS * _sp(lpl)
        v = 5 - lpl
        out[li] = np.maximum(v, 0)
        bar[li] = np.where(v > -lb, lb + _sp(v), 0.0)
        mag[li] = np.where(v > -lb, 5 + np.abs(lpl), 0.0)
    return out, bar, mag


def _bp_check(model, batch, t_values, seed, ck):
    K = model.num_classes
    bl, B, n_all, gen = _common(batch)
    n, R = bl.shape[0], len(t_values)
    pn, tu = synthetic.make_bp_noise(R, n, seed=seed)
    tu = _crafted_u(tu, model, t_values)
    loss, res = model.eval_losses(to_dev(batch), t_values, pos_noise=pn, type_uniform=tu)
    x0, v0 = _np(batch['ligand_pos']), batch['ligand_atom_type'].numpy()
    prot, bp = _np(batch['protein_pos']), batch['protein_element_batch'].numpy()
    reps, bars, scales = [], [], []
    for r, t in enumerate(t_values):
        cf = model.eval_coef(t)
        eps, u = _np(pn[r]), tu[r].numpy()
        # the absorbing-state mask, exactly
        mask = gen & (u < np.float32(cf.mask_prob))
        assert np.array_equal(res[r]['mask_gen'].cpu().numpy(), mask), f't={t}: type mask differs'
        assert torch.equal(res[r]['vt'].cpu(), torch.nn.functional.one_hot(torch.from_numpy(np.where(mask, 0, v0)), K).float())
        # zero-centred noise target and its graph mean (the CoM target)
        cnt_all = np.maximum(n_all, 1)
        mean = np.stack([np.bincount(bl, eps[:, c], minlength=B) for c in range(3)], 1) / cnt_all[:, None]
        depth = (np.ceil(n_all / 128) + 8)[:, None]
        mean_b = depth * U32 * np.stack([np.bincount(bl, np.abs(eps[:, c]), minlength=B) for c in range(3)], 1) / \
            cnt_all[:, None] + _sp(mean)
        e0, c0 = _np(res[r]['eps_0']), _np(res[r]['eps_0_com'])
        ck('eps_0', e0, eps - mean[bl], mean_b[bl] + _sp(eps - mean[bl]), min_tight=0.9, scale=np.abs(eps) + np.abs(mean[bl]))
        ck('eps_0_com', c0, mean[bl], mean_b[bl], min_tight=0.9, scale=1.0)
        ep, cp = _np(res[r]['eps_pred']), _np(res[r]['eps_pred_com'])
        pos_e, com_e = ((ep - e0) ** 2).sum(1), ((cp - c0) ** 2).sum(1)
        # masked-type cross-entropy on the probabilities
        pr = _np(res[r]['c_pred'])
        m2 = pr.max(1)
        ls = np.log(np.exp(pr - m2[:, None]).sum(1))
        ce = -(pr[np.arange(n), v0] - m2 - ls)
        ce_b = ULPS * (_sp(m2) + _sp(ls) + _sp(ce) + K * U32)
        # posterior mean x_s from the rebuilt x_t, then the interior loss
        sa, sig = math.sqrt(cf.alphas_cumprod), math.sqrt(1.0 - cf.alphas_cumprod)
        xt = np.where(gen[:, None], sa * x0 + sig * eps, x0)
        bs = cf.beta * (-(ep + cp) / sig)
        xs = np.where(gen[:, None], (xt + bs) / math.sqrt(1.0 - cf.beta), xt)
        xs_b = ULPS * (_sp(sa * x0) + _sp(sig * eps) + _sp(xt) + _sp(bs) + _sp(xs))
        inter, inter_b, inter_m = _bp_inter(xs, xs_b, prot, bl, bp, B)
        row = []
        for e, b, sel, empty in ((pos_e, ULPS * _sp(pos_e), gen, math.nan), (ce, ce_b, mask, 0.0),
                                 (com_e, ULPS * _sp(com_e), gen, math.nan)):
            gm, gb, cnt = _graph_mean(e, b, sel, bl, n_all, B)
            last = int(np.nonzero(cnt)[0].max()) if cnt.any() else -1
            v, vb = _rows_mean(gm, gb, last)
            row.append((empty, 0.0) if last < 0 else (v, vb))
        row.append((inter.sum() / n, inter_b.sum() / n + (np.ceil(n_all.max() / 128) + 8 + B) * U32 * inter.mean()))
        reps.append([v for v, _ in row])
        bars.append([b for _, b in row])
        scales.append(inter_m.mean())
    reps, bars = np.array(reps), np.array(bars)
    rep = _np(model.last_rep_loss)
    assert rep.shape == (R, 4)
    for i, k in enumerate(('pos', 'atom', 'com', 'inter')):
        ck(f'per-t {k}', rep[:, i], reps[:, i], bars[:, i], scale=np.array(scales) if k == 'inter' else 0.0)
        assert torch.equal(loss[k], torch.mean(model.last_rep_loss[:, i].cpu())) or \
            (math.isnan(float(loss[k])) and bool(model.last_rep_loss[:, i].isnan().any())), f'{k}: mean over t differs'
    return loss


@pytest.mark.gpu
@pytest.mark.parametrize('K', KS)
@pytest.mark.parametrize('layout', BP_LAYOUTS)
def test_diffbp_loss_against_float64(layout, K):
    ck = Checks(f'diffbp {layout} K={K}')
    loss = _bp_check(_model('bp', K), _batch(layout, K, seed=21), T_TD, seed=22, ck=ck)
    if layout == 'nothing_generated':
        assert math.isnan(float(loss['pos'])) and math.isnan(float(loss['com']))
        assert float(loss['atom']) == 0.0                 # the type mask is gen-gated: nothing masked
    ck.report()


@pytest.mark.gpu
def test_diffbp_atom_loss_is_zero_without_masked_atoms():
    model = _model('bp', 13)
    batch = _batch('sizes', 13, seed=23)
    pn, tu = synthetic.make_bp_noise(1, batch['ligand_pos'].shape[0], seed=24)
    loss, res = model.eval_losses(to_dev(batch), [0], pos_noise=pn, type_uniform=tu)   # t = 0: mask probability 0
    assert not bool(res[0]['mask_gen'].any())
    assert float(loss['atom']) == 0.0 and math.isfinite(float(loss['pos']))


# ---- DiffSBDD ---------------------------------------------------------------------------------------------------------

def _cdf_diff(hi, lo):
    """Phi(hi) - Phi(lo) in float64 without cancellation in either tail."""
    upper = 0.5 * (erfc(lo * SQRT1_2) - erfc(hi * SQRT1_2))          # both tails above 0
    lower = 0.5 * (erfc(-hi * SQRT1_2) - erfc(-lo * SQRT1_2))        # both below 0
    mid = 1.0 - 0.5 * erfc(-lo * SQRT1_2) - 0.5 * erfc(hi * SQRT1_2)
    return np.where(lo >= 0, upper, np.where(hi <= 0, lower, mid))


def _pdf(x):
    return np.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def _ng0_terms(cf, K):
    """The six terms of a graph without ligand atoms (d = -3, -K), in the kernel's fp32 operation order."""
    f = np.float32
    dp, dc = f(-3), f(-K)
    return np.array([f(f(cf.pos_t_weight) * f(0)),
                     f(f(f(0.5) * f(0)) - f(dp * f(cf.pos_log_const))),
                     f(f(f(dp * f(cf.pos_log_inv_sigma_T)) + f(f(0.5) * f(f(dp * f(cf.pos_sigma2_T)) + f(0))))
                       - f(f(0.5) * dp)),
                     f(f(cf.type_t_weight) * f(0)),
                     f(f(-f(0)) - f(dc * f(cf.type_log_const))),
                     f(f(f(cf.type_log_inv_sigma_T) + f(f(0.5) * f(f(cf.type_sigma2_T) + f(0)))) - f(0.5))])


def _sbdd_check(model, batch, t_values, seed, ck, with_pos0):
    K = model.num_classes
    bl, B_all, n_all, gen = _common(batch)
    n, R = bl.shape[0], len(t_values)
    noise = synthetic.make_sbdd_eval_noise(R, n, K, seed=seed)
    loss, res = model.eval_losses(to_dev(batch), t_values, noise=noise)
    terms = _np(model.last_terms)
    B = int(bl.max()) + 1
    assert terms.shape == (R, B, 6)
    x0, v0 = _np(batch['ligand_pos']), batch['ligand_atom_type'].numpy()
    hot = np.arange(K)[None] == v0[:, None]
    c0 = hot * 0.25
    reps, rep_b, rep_s, per_t32 = [], [], [], []
    for j, t in enumerate(t_values):
        cf = model.eval_coef(t)
        ext, ect, ex0, ec0 = (_np(noise[k][j]) for k in ('x_t', 'c_t', 'x_0', 'c_0'))
        xp_t, cp = _np(res[j]['eps_pred_pos']), _np(res[j]['eps_pred_atom'])
        want, bar, scale = np.zeros((B, 6)), np.zeros((B, 6)), np.zeros((B, 6))
        for g in range(B):
            a = np.nonzero(bl == g)[0]
            ng = a.size
            if ng == 0:
                assert np.array_equal(terms[j, g], _ng0_terms(cf, K)), f't={t} graph {g}: n_g = 0 terms differ'
                want[g], bar[g] = terms[j, g], 0.0
                continue
            depth = math.ceil(ng / 128) + 8
            X0, G = x0[a], gen[a]
            mean0 = X0.mean(0)
            err_mean0 = depth * U32 * np.abs(X0).mean(0) + _sp(mean0)
            x0c = X0 - mean0
            err_x0c = _sp(X0) + _sp(x0c) + err_mean0
            dp, dc = 3.0 * (ng - 1), float(K * (ng - 1))

            def gsum(e, eb):
                return e.sum(), eb.sum() + depth * U32 * np.abs(e).sum()
            # pos_t
            d = ext[a] - xp_t[a]
            et = (d * d).sum(1)
            S, Sb = gsum(et, ULPS * _sp(et))
            want[g, 0], bar[g, 0] = cf.pos_t_weight * S, abs(cf.pos_t_weight) * Sb + ULPS * _sp(cf.pos_t_weight * S)
            # pos_0: the t = 0 copy's prediction is its noised input position
            if with_pos0:
                xn = cf.pos_alpha_0 * x0c + cf.pos_sigma_0 * ex0[a]
                m = xn.mean(0)
                xp0 = np.where(G[:, None], xn - m, x0c)
                err_xp0 = np.where(G[:, None], cf.pos_alpha_0 * err_x0c + ULPS * (_sp(cf.pos_alpha_0 * x0c)
                                   + _sp(cf.pos_sigma_0 * ex0[a]) + _sp(xn) + _sp(xn - m)) + depth * U32 * np.abs(xn).mean(0)
                                   + _sp(m), err_x0c)
                d0 = ex0[a] - xp0
                e0 = (d0 * d0).sum(1)
                S, Sb = gsum(e0, ULPS * _sp(e0) + 2 * (np.abs(d0) * err_xp0).sum(1))
                want[g, 1] = 0.5 * S - dp * cf.pos_log_const
                bar[g, 1] = 0.5 * Sb + ULPS * (_sp(0.5 * S) + _sp(dp * cf.pos_log_const) + _sp(want[g, 1]))
                scale[g, 1] = 0.5 * S + abs(dp * cf.pos_log_const)
            # pos_kl
            xa = cf.pos_alpha_T * x0c
            mu = (xa * xa).sum(1)
            S, Sb = gsum(mu, ULPS * _sp(mu) + 2 * cf.pos_alpha_T * (np.abs(xa) * err_x0c).sum(1))
            want[g, 2] = dp * cf.pos_log_inv_sigma_T + 0.5 * (dp * cf.pos_sigma2_T + S) - 0.5 * dp
            bar[g, 2] = 0.5 * Sb + ULPS * (_sp(dp * cf.pos_log_inv_sigma_T) + _sp(dp * cf.pos_sigma2_T) + _sp(S)
                                           + _sp(0.5 * dp) + _sp(want[g, 2]))
            scale[g, 2] = abs(dp * cf.pos_log_inv_sigma_T) + 0.5 * (dp * cf.pos_sigma2_T + S) + 0.5 * dp
            # atom_t
            da = ect[a] - cp[a]
            ea = (da * da).sum(1)
            S, Sb = gsum(ea, ULPS * _sp(ea) + K * U32 * ea)
            want[g, 3], bar[g, 3] = cf.type_t_weight * S, abs(cf.type_t_weight) * Sb + ULPS * _sp(cf.type_t_weight * S)
            # atom_0: discretised likelihood of the t = 0 copy's noised types, bounded by its conditioning in the tails
            ac, sc = cf.type_alpha_0, cf.type_sigma_0
            cz = np.where(G[:, None], ac * c0[a] + sc * ec0[a], c0[a])
            cz_b = np.where(G[:, None], ULPS * (_sp(ac * c0[a]) + _sp(sc * ec0[a]) + _sp(cz)), 0.0)
            cen = 4 * cz - 1
            s0 = sc * 4
            hi, lo = (cen + 0.5) / s0, (cen - 0.5) / s0
            arg_b = (4 * cz_b + ULPS * (_sp(cen) + U32)) / s0 + ULPS * (_sp(hi) + _sp(lo))
            pr = _cdf_diff(hi, lo)
            pr_b = 2 * ULPS * U32 + (_pdf(hi) + _pdf(lo)) * arg_b
            lp = np.log(pr + 1e-10)
            lp_b = pr_b / (pr + 1e-10) + ULPS * _sp(lp)
            mx = lp.max(1, keepdims=True)
            w = np.exp(lp - mx)
            lse = (mx + np.log(w.sum(1, keepdims=True)))[:, 0]
            logp = lp[np.arange(ng), v0[a]] - lse
            logp_b = lp_b[np.arange(ng), v0[a]] + (w / w.sum(1, keepdims=True) * lp_b).sum(1) + ULPS * (_sp(lse) + K * U32)
            S, Sb = gsum(logp, logp_b)
            want[g, 4] = -S - dc * cf.type_log_const
            bar[g, 4] = Sb + ULPS * (_sp(S) + _sp(dc * cf.type_log_const) + _sp(want[g, 4]))
            scale[g, 4] = abs(S) + abs(dc * cf.type_log_const)
            # atom_kl (d = 1)
            Sca = ng * (cf.type_alpha_T * 0.25) ** 2
            want[g, 5] = cf.type_log_inv_sigma_T + 0.5 * (cf.type_sigma2_T + Sca) - 0.5
            bar[g, 5] = depth * U32 * Sca + ULPS * (_sp(cf.type_log_inv_sigma_T) + _sp(cf.type_sigma2_T) + _sp(Sca)
                                                    + _sp(want[g, 5]) + _sp(0.5))
            scale[g, 5] = abs(cf.type_log_inv_sigma_T) + 0.5 * (cf.type_sigma2_T + Sca) + 0.5
        names = ('pos_t', 'pos_0', 'pos_kl', 'atom_t', 'atom_0', 'atom_kl')
        for i, name in enumerate(names):
            if i == 1 and not with_pos0:
                continue
            ck(name, terms[j, :, i], want[:, i], bar[:, i], scale=scale[:, i])
        # the per-t loss over the B rows, exactly from the terms and against float64
        t32 = terms[j].astype(np.float32)
        per = []
        for lo_, name in ((0, 'pos'), (3, 'atom')):
            s = np.float32(0)
            for g in range(B):
                s = np.float32(s + np.float32(np.float32(t32[g, lo_] + t32[g, lo_ + 1]) + t32[g, lo_ + 2]))
            per.append(np.float32(s / np.float32(B)))
        per_t32.append(per)
        if with_pos0:
            reps.append([want[:, :3].sum(1).mean(), want[:, 3:].sum(1).mean()])
            rep_b.append([bar[:, :3].sum(1).mean(), bar[:, 3:].sum(1).mean()])
            mag = np.maximum(np.abs(want), scale)
            rep_s.append([mag[:, :3].sum(1).mean(), mag[:, 3:].sum(1).mean()])
    for i, k in enumerate(('pos', 'atom')):
        assert torch.equal(loss[k], torch.mean(torch.tensor([float(v[i]) for v in per_t32]))), f'{k}: per-t reduction differs'
    if with_pos0:
        reps, rep_b, rep_s = np.array(reps), np.array(rep_b), np.array(rep_s)
        for i, k in enumerate(('pos', 'atom')):
            ck(f'loss {k}', float(loss[k]), reps[:, i].mean(), rep_b[:, i].mean() + (B + R + 6) * U32 * rep_s[:, i].mean(),
               scale=rep_s[:, i].mean())
    return loss


@pytest.mark.gpu
@pytest.mark.parametrize('K', KS)
@pytest.mark.parametrize('layout', list(LAYOUTS))
def test_diffsbdd_terms_against_float64(layout, K):
    ck = Checks(f'diffsbdd {layout} K={K}')
    _sbdd_check(_model('sbdd', K), _batch(layout, K, seed=31), T_SBDD, seed=32, ck=ck, with_pos0=True)
    ck.report()


@pytest.mark.gpu
def test_diffsbdd_seeded_coordinate_head_five_terms():
    """With a moving t = 0 copy its prediction is not returned: the other five terms still match float64."""
    ck = Checks('diffsbdd seeded xv_func sizes K=13')
    _sbdd_check(_model('sbdd_xv', 13), _batch('sizes', 13, seed=33), T_SBDD, seed=34, ck=ck, with_pos0=False)
    ck.report()


# ---- determinism at the large layouts ---------------------------------------------------------------------------------

def _flat(loss, res, extra):
    out = [loss[k] for k in loss] + [v for r in res for v in r.values()] + [extra]
    return [t.cpu().clone() for t in out]


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ('td', 'bp', 'sbdd'))
def test_large_layouts_are_bit_identical(kind):
    """Repeated calls, and a split into one launch per timestep, are bit-identical to one launch."""
    model = _model(kind, 16)
    batch = to_dev(_batch('lig1500', 16, seed=41))
    n, R, K = batch['ligand_pos'].shape[0], 4, 16
    n_nodes = n + batch['protein_pos'].shape[0]
    if kind == 'sbdd':
        noise = synthetic.make_sbdd_eval_noise(R, n, K, seed=42)
        run = lambda **kw: _flat(*model.eval_losses(batch, T_SBDD, noise=noise, **kw), model.last_terms)
        split = 2 * n_nodes                               # a timestep counts twice
    else:
        pn, tu = (synthetic.make_noise(R, n, K, seed=42) if kind == 'td' else synthetic.make_bp_noise(R, n, seed=42))
        extra = (lambda: model.last_graph_loss) if kind == 'td' else (lambda: torch.zeros(1))
        run = lambda **kw: _flat(*model.eval_losses(batch, T_TD, pos_noise=pn, type_uniform=tu, **kw), extra())
        split = n_nodes
    one = run()
    launches = model.last_launches
    for other in (run(), run(max_nodes=split)):
        assert len(other) == len(one)
        for a, b in zip(one, other):
            assert torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan())
                                         and torch.equal(a[~a.isnan()], b[~b.isnan()]))
    assert model.last_launches > launches                  # the split ran more launches
