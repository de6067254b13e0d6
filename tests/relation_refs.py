"""Float64 reference of the cond=relation logit adjustment: `relation_num_update` SGD steps on the bin log-probabilities for
the mean over (layout, cost function) of the 14 relation costs, evaluated on the expected boxes (softmax over each
attribute's bins times the bin centres; node 0 is the canvas).  The costs are written from their definitions as float64
torch expressions and the gradient comes from torch.autograd: nothing here shares the hand-derived gradient of the kernel
(relation.cuh) or of the oracle (O.relation_cost_and_grad).

ReLU terms.  Every cost is a sum of terms  relu(cI * Q_I[i] + cJ * Q_J[j] + k)  over the edges i -> j whose edge_attr has
the term's bit, both ends valid (not PAD), with the source either an element or the canvas.  Q is one of the box
quantities area = w h, y, l = x - w/2, t = y - h/2, r = x + w/2, b = y + h/2.  `less(a, b)` = relu(a - b + 1e-8) and
`less_equal(a, b)` = relu(a - b).  The left / right / center costs also carry the two vertical-overlap terms, kept apart per
code so that each kernel branch has a term of its own.

fp32 error model of one update (u = 2^-24; x_k = v_k - max_k v_k is the shifted bin log-prob):
  p_k      relative error  (|x_k| + 10) u        (v - m rounded, expf <= 2 ulp, a 32-lane tree sum, the division)
  box      |d| <= sum_k p_k |c_k| (eps_p_k + 6 u)  (the products and the 32-lane tree sum)
  g        d(sum of costs) / d(box): x and y are sums of +-1 (exact); w and h carry the area coefficients +-0.9f, +-1.1f, +-1,
           accumulated in fp32, and the box error of the other side: (n_a + 1) 1.1 n_a u |h| + |g_area| d_h + 2 u (|g_area h| + |g_w|)
           with n_a the node's active size terms
  update   |d Delta| <= step (|g| p (|c - b| (eps_p + 6 u) + d_box) + p |c - b| d_g),  step = lambda / (batch_total 14)
  store    + u |v_new|
A term's argument carries the box errors of its operands plus 4 u of its operands' magnitudes; where |arg| is within that
bound of 0 the branch the kernel takes is not determined by the arithmetic (a kink)."""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

from oracle import layoutdm_oracle as O

U32 = 2.0 ** -24
EPS = 1e-8
AL, AH = 0.9, 1.1
N_FUNCS = 14
LOC_L, LOC_T, LOC_R, LOC_B, LOC_C = 5, 6, 7, 8, 9

# (name, bit, source, cI, Q_I, cJ, Q_J, k)
TERMS: List[Tuple[str, int, str, float, Optional[str], float, str, float]] = []
TERMS += [("size_sm", 1, "any", -AL, "area", 1.0, "area", 0.0),                       # a_j <= 0.9 a_i
          ("size_eq_lo", 2, "any", AL, "area", -1.0, "area", EPS),                    # 0.9 a_i < a_j
          ("size_eq_hi", 2, "any", -AH, "area", 1.0, "area", EPS),                    # a_j < 1.1 a_i
          ("size_lg", 3, "any", AH, "area", -1.0, "area", 0.0),                       # 1.1 a_i <= a_j
          ("canvas_top", LOC_T, "canvas", 0.0, None, 1.0, "y", -1.0 / 3),             # y_j <= 1/3
          ("canvas_center_lo", LOC_C, "canvas", 0.0, None, -1.0, "y", 1.0 / 3 + EPS),  # 1/3 < y_j
          ("canvas_center_hi", LOC_C, "canvas", 0.0, None, 1.0, "y", -2.0 / 3 + EPS),  # y_j < 2/3
          ("canvas_bottom", LOC_B, "canvas", 0.0, None, -1.0, "y", 2.0 / 3),           # 2/3 <= y_j
          ("top", LOC_T, "elem", -1.0, "t", 1.0, "b", 0.0),                           # b_j <= t_i
          ("bottom", LOC_B, "elem", 1.0, "b", -1.0, "t", 0.0),                        # b_i <= t_j
          ("left", LOC_L, "elem", -1.0, "l", 1.0, "r", 0.0),                          # r_j <= l_i
          ("right", LOC_R, "elem", 1.0, "r", -1.0, "l", 0.0),                         # r_i <= l_j
          ("center_lo", LOC_C, "elem", 1.0, "l", -1.0, "r", EPS),                     # l_i < r_j
          ("center_hi", LOC_C, "elem", -1.0, "r", 1.0, "l", EPS)]                     # l_j < r_i
for _code, _nm in ((LOC_L, "left"), (LOC_R, "right"), (LOC_C, "center")):
    TERMS += [(f"{_nm}_vov_lo", _code, "elem", 1.0, "t", -1.0, "b", EPS),             # t_i < b_j
              (f"{_nm}_vov_hi", _code, "elem", -1.0, "b", 1.0, "t", EPS)]             # t_j < b_i
TERM_NAMES = [t[0] for t in TERMS]


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def linear_centers32(n_bins: int) -> torch.Tensor:
    return torch.stack([torch.as_tensor(c, dtype=torch.float32) for c in O.linear_centers(n_bins)])


def canvas_box(centers: torch.Tensor, n_bins: int) -> torch.Tensor:
    """the canvas node's box: the centre of the bin that encodes (0.5, 0.5, 1, 1), by the linear rule when the centres are the
    linear ones and by the nearest centre otherwise (the rule O.relation_bbox follows).  float64 (4,)"""
    lin = linear_centers32(n_bins)
    v = torch.tensor([0.5, 0.5, 1.0, 1.0], dtype=torch.float64)
    if torch.equal(centers, lin):
        d = 1.0 / n_bins
        q = torch.cat([v[:2].clamp(0.0, 1.0 - d), v[2:].clamp(d, 1.0) - d])
        bins = torch.round(n_bins * q).long()
    else:
        bins = (centers.double() - v[:, None]).pow(2).argmin(dim=1)
    return centers.double()[torch.arange(4), bins]


def bin_logprobs(lp: torch.Tensor, vo: O.VocabSpec) -> torch.Tensor:
    """(B,S,C) -> (B,E,4,n_bins): the log-probs of each element's attribute a over attribute a's own bins"""
    B, A, nb, nc = lp.shape[0], vo.n_attr, vo.n_bins, vo.n_cat
    return torch.stack([lp[:, a + 1::A, nc + a * nb: nc + (a + 1) * nb] for a in range(4)], dim=2)


def put_bins(lp: torch.Tensor, v: torch.Tensor, vo: O.VocabSpec) -> torch.Tensor:
    out = lp.clone()
    A, nb, nc = vo.n_attr, vo.n_bins, vo.n_cat
    for a in range(4):
        out[:, a + 1::A, nc + a * nb: nc + (a + 1) * nb] = v[:, :, a].to(out.dtype)
    return out


def valid_nodes(cond_seq: torch.Tensor, vo: O.VocabSpec) -> torch.Tensor:
    B = cond_seq.shape[0]
    return torch.cat([torch.ones(B, 1, dtype=torch.bool), cond_seq[:, ::vo.n_attr] != vo.pad_id], dim=1)


# ---------------------------------------------------------------------------------------------------------------------
# costs
# ---------------------------------------------------------------------------------------------------------------------
def quantities(box: torch.Tensor) -> Dict[str, torch.Tensor]:
    x, y, w, h = box.unbind(-1)
    return {"area": w * h, "y": y, "l": x - w / 2, "t": y - h / 2, "r": x + w / 2, "b": y + h / 2}


def term_masks(adj: torch.Tensor, valid: torch.Tensor) -> List[torch.Tensor]:
    """per term: (B,N,N) bool, the edges i -> j the term applies to"""
    N = adj.shape[1]
    both = valid[:, :, None] & valid[:, None, :]
    src_canvas = (torch.arange(N) == 0)[None, :, None].expand_as(both)
    out = []
    for name, bit, src, *_ in TERMS:
        m = ((adj.long() >> bit) & 1).bool() & both
        out.append(m if src == "any" else m & (src_canvas if src == "canvas" else ~src_canvas))
    return out


def term_args(q: Dict[str, torch.Tensor], mutate: Optional[Tuple[int, str]] = None) -> List[torch.Tensor]:
    """per term: its argument (B,N,N), [b, i, j] for the edge i -> j.  mutate = (term index, "drop_i" / "drop_j") cuts the
    gradient to one end of that term (a kernel branch that misses one of its two nodes)"""
    out = []
    for n, (name, bit, src, cI, QI, cJ, QJ, k) in enumerate(TERMS):
        qj = q[QJ]
        qi = q[QI] if QI is not None else None
        if mutate is not None and mutate[0] == n:
            if mutate[1] == "drop_i" and qi is not None:
                qi = qi.detach()
            if mutate[1] == "drop_j":
                qj = qj.detach()
        a = cJ * qj[:, None, :] + k
        if qi is not None:
            a = a + cI * qi[:, :, None]
        out.append(a)
    return out


def total_cost(box, masks, force=None, mutate=None):
    """sum over layouts of the sum of the 14 costs.  force: per term None or a (B,N,N) int tensor, -1 = relu, 0 = branch
    off, 1 = branch on.  mutate = (term index, "drop" / "flip" / "drop_i" / "drop_j")."""
    args = term_args(quantities(box), mutate if mutate and mutate[1] in ("drop_i", "drop_j") else None)
    cost = box.new_zeros(())
    for n, (a, m) in enumerate(zip(args, masks)):
        r = torch.relu(a)
        if force is not None and force[n] is not None:
            r = torch.where(force[n] == 1, a, torch.where(force[n] == 0, torch.zeros_like(a), r))
        r = torch.where(m, r, torch.zeros_like(r))
        if mutate is not None and mutate[0] == n:
            if mutate[1] == "drop":
                continue
            if mutate[1] == "flip":
                r = -r
        cost = cost + r.sum()
    return cost


def expected_boxes(v: torch.Tensor, centers64: torch.Tensor, cbox: torch.Tensor):
    """v (B,E,4,nb) float64 bin log-probs -> p (B,E,4,nb), box (B,N,4) with node 0 the canvas"""
    p = torch.softmax(v, dim=-1)
    be = (p * centers64[None, None]).sum(-1)
    box = torch.cat([cbox[None, None].expand(v.shape[0], 1, 4), be], dim=1)
    return p, box


# ---------------------------------------------------------------------------------------------------------------------
# update, term table, gate
# ---------------------------------------------------------------------------------------------------------------------
class Problem:
    """one relation update problem: the log-probs the update starts from and everything it depends on"""

    def __init__(self, lp: torch.Tensor, cond_seq: torch.Tensor, adj: torch.Tensor, centers: Optional[torch.Tensor],
                 vo: O.VocabSpec, lam: float, batch_total: Optional[int] = None):
        self.vo = vo
        self.lp = lp
        self.v0 = bin_logprobs(lp.double(), vo)
        self.valid = valid_nodes(cond_seq, vo)
        self.adj = adj
        c32 = linear_centers32(vo.n_bins) if centers is None else centers.float()
        self.cen = c32.double()
        self.cbox = canvas_box(c32, vo.n_bins)
        self.masks = term_masks(adj, self.valid)
        self.step = lam / ((batch_total or lp.shape[0]) * N_FUNCS)
        self.elem_valid = self.valid[:, 1:, None, None]

    def grad(self, v, force=None, mutate=None):
        v = v.detach().requires_grad_(True)
        _, box = expected_boxes(v, self.cen, self.cbox)
        cost = total_cost(box, self.masks, force, mutate)
        if not cost.requires_grad:
            return torch.zeros_like(v)
        (g,) = torch.autograd.grad(cost, v)
        return g

    def run(self, n_update: int, force=None, mutate=None, perturb: Optional[Callable] = None, record: Optional[list] = None):
        """n_update SGD steps from the problem's log-probs -> float64 bin log-probs (B,E,4,nb).  Only valid elements move.
        perturb(u, v, v_new) -> v_new after each update; record gets each update's term activity"""
        v = self.v0.clone()
        for u in range(n_update):
            if record is not None:
                record.append(self.table(v)["active"])
            g = self.grad(v, force if u == 0 else None, mutate)
            v_new = torch.where(self.elem_valid, v - self.step * g, v)
            if perturb is not None:
                v_new = perturb(u, v, v_new)
            v = v_new
        return v

    def table(self, v=None) -> dict:
        """the ReLU term table at the state v: per term the argument (B,N,N), whether the term applies (edge bit, valid ends,
        source kind) and is active (> 0), and the bound on the argument's fp32 error"""
        v = self.v0 if v is None else v
        with torch.no_grad():
            p, box = expected_boxes(v, self.cen, self.cbox)
            dbox = self.box_error(v, p)
            q = quantities(box)
            x, y, w, h = box.unbind(-1)
            dx, dy, dw, dh = dbox.unbind(-1)
            dq = {"area": dw * h.abs() + w.abs() * dh + U32 * (w * h).abs(), "y": dy,
                  "l": dx + dw / 2 + 2 * U32 * (x.abs() + w.abs() / 2), "r": dx + dw / 2 + 2 * U32 * (x.abs() + w.abs() / 2),
                  "t": dy + dh / 2 + 2 * U32 * (y.abs() + h.abs() / 2), "b": dy + dh / 2 + 2 * U32 * (y.abs() + h.abs() / 2)}
            args = term_args(q)
            err = []
            for (name, bit, src, cI, QI, cJ, QJ, k) in TERMS:
                e = abs(cJ) * dq[QJ][:, None, :] + 4 * U32 * (abs(cJ) * q[QJ].abs()[:, None, :] + abs(k)) + U32
                if QI is not None:
                    e = e + abs(cI) * dq[QI][:, :, None] + 4 * U32 * abs(cI) * q[QI].abs()[:, :, None]
                err.append(e)
        active = [m & (a > 0) for a, m in zip(args, self.masks)]
        return {"arg": args, "applies": self.masks, "active": active, "err": err}

    def box_error(self, v, p=None):
        """(B,N,4) bound on the fp32 expected box's error; the canvas box is a centre value, exact"""
        p = torch.softmax(v, dim=-1) if p is None else p
        xs = (v - v.amax(-1, keepdim=True)).abs()
        eps_p = (xs + 10) * U32
        db = (p * self.cen.abs()[None, None] * (eps_p + 6 * U32)).sum(-1)
        return torch.cat([torch.zeros_like(db[:, :1]), db], dim=1)

    def gate(self, v=None, parts=False):
        """(B,E,4,nb) bound on |fp32 update - float64 update| of one update from the state v (see the module docstring);
        parts: (the update's share, the store's share) instead of their sum"""
        v = self.v0 if v is None else v
        vv = v.detach().requires_grad_(True)
        p, box = expected_boxes(vv, self.cen, self.cbox)
        boxl = box.detach().requires_grad_(True)
        q = quantities(boxl)
        cost = total_cost_from_q(q, self.masks)
        gb, ga = torch.autograd.grad(cost, [boxl, q["area"]], allow_unused=True) if cost.requires_grad else (None, None)
        gb = torch.zeros_like(boxl) if gb is None else gb
        ga = torch.zeros_like(q["area"]) if ga is None else ga
        p, box = p.detach(), box.detach()
        tab = self.table(v)
        n_a = torch.zeros_like(ga)
        for n, (name, *_r) in enumerate(TERMS):
            if name.startswith("size"):
                act = tab["active"][n].double()
                n_a += act.sum(2) + act.sum(1)
        dbox = self.box_error(v, p)
        x, y, w, h = box.unbind(-1)
        dg = torch.zeros_like(gb)
        acc = (n_a + 1) * AH * n_a * U32
        dg[..., 2] = acc * h.abs() + ga.abs() * dbox[..., 3] + 2 * U32 * ((ga * h).abs() + gb[..., 2].abs())
        dg[..., 3] = acc * w.abs() + ga.abs() * dbox[..., 2] + 2 * U32 * ((ga * w).abs() + gb[..., 3].abs())
        g, dg, db, bx = gb[:, 1:, :, None], dg[:, 1:, :, None], dbox[:, 1:, :, None], box[:, 1:, :, None]
        cmb = (self.cen[None, None] - bx).abs()
        eps_p = ((v - v.amax(-1, keepdim=True)).abs() + 10) * U32
        d_delta = self.step * (g.abs() * p * (cmb * (eps_p + 6 * U32) + db) + p * cmb * dg)
        v_new = v - self.step * g * p * (self.cen[None, None] - bx)
        d_delta = torch.where(self.elem_valid, d_delta, torch.zeros_like(d_delta)).detach()
        store = torch.where(self.elem_valid, U32 * v_new.abs(), U32 * v.abs()).detach()
        return (d_delta, store) if parts else d_delta + store


def total_cost_from_q(q, masks):
    cost = q["y"].new_zeros(())
    for a, m in zip(term_args(q), masks):
        cost = cost + torch.where(m, torch.relu(a), torch.zeros_like(a)).sum()
    return cost


def kinks(tab: dict) -> List[Tuple[int, int, int, int]]:
    """(term, b, i, j) of every applying term whose argument lies within its fp32 error bound of 0"""
    out = []
    for n, (a, m, e) in enumerate(zip(tab["arg"], tab["applies"], tab["err"])):
        idx = (m & (a.abs() <= e)).nonzero().tolist()
        out += [(n, b, i, j) for b, i, j in idx]
    return out


def kink_variants(prob: Problem, kk: Sequence[Tuple[int, int, int, int]], max_per_layout: int = 4):
    """force patterns that take every combination of branches at the ambiguous terms of each layout, batch-wide: variant k
    forces the i-th ambiguous term of every layout on when bit i of k is set.  -> list of force lists (None: no kinks)"""
    per = {}
    for n, b, i, j in kk:
        per.setdefault(b, []).append((n, i, j))
    if not per:
        return [None]
    kmax = max(len(x) for x in per.values())
    assert kmax <= max_per_layout, f"{kmax} ambiguous ReLU terms in one layout: the inputs are too close to the kinks"
    B, N = prob.adj.shape[0], prob.adj.shape[1]
    out = []
    for k in range(2 ** kmax):
        f = [None] * len(TERMS)
        for b, lst in per.items():
            for bit, (n, i, j) in enumerate(lst):
                if f[n] is None:
                    f[n] = torch.full((B, N, N), -1, dtype=torch.long)
                f[n][b, i, j] = (k >> bit) & 1
        out.append(f)
    return out


def coverage(tabs: Sequence[dict]) -> Dict[str, Tuple[int, int]]:
    """per term: (applying edges where it is active, applying edges where it is inactive), summed over the tables"""
    out = {}
    for n, name in enumerate(TERM_NAMES):
        on = sum(int((t["applies"][n] & (t["arg"][n] > 0)).sum()) for t in tabs)
        off = sum(int((t["applies"][n] & ~(t["arg"][n] > 0)).sum()) for t in tabs)
        out[name] = (on, off)
    return out


def multi_update_gate(prob: Problem, n_up: int, draws: int = 4, seed: int = 0):
    """several updates: the reference output, its gate (B,E,4,nb) and the well-conditioned layouts (B,).  Every update of
    `draws` reruns is perturbed by a uniform draw within that update's gate; the gate is 4x the spread of the reruns (per
    element and attribute) plus the last update's own gate.  A layout is well conditioned when no rerun changes a ReLU
    branch in any update and the unperturbed trajectory meets no kink."""
    rec = []
    ref = prob.run(n_up, record=rec)
    ok = torch.ones(ref.shape[0], dtype=torch.bool)
    v = prob.v0
    for u in range(n_up):
        for n, b, i, j in kinks(prob.table(v)):
            ok[b] = False
        if u < n_up - 1:
            v = prob.run(u + 1)
    last_gate = prob.gate(v)
    g = torch.Generator().manual_seed(seed)
    spread = torch.zeros_like(ref)

    def perturb(u, v0, v1):
        return v1 + (2 * torch.rand(v1.shape, generator=g, dtype=torch.float64) - 1) * prob.gate(v0)

    for _ in range(draws):
        rd = []
        out = prob.run(n_up, perturb=perturb, record=rd)
        for a_ref, a_d in zip(rec, rd):
            for m0, m1 in zip(a_ref, a_d):
                ok &= (m0 == m1).flatten(1).all(1)
        spread = torch.maximum(spread, (out - ref).abs())
    return ref, 4 * spread.amax(-1, keepdim=True) + last_gate, ok


# ---------------------------------------------------------------------------------------------------------------------
# designed batches (the GPU test's cases)
# ---------------------------------------------------------------------------------------------------------------------
VOCABS = {"rico25": O.RICO25, "n_cat10_n_bins30": O.VocabSpec(n_cat=10, n_bins=30),
          "n_cat3_n_bins31": O.VocabSpec(n_cat=3, n_bins=31), "n_elem20": O.VocabSpec(n_elem=20)}
CENTERS = ("none", "linear", "kmeans")


def one_update_case(vname: str, lam: float) -> Tuple[int, int]:
    """(B, seed) of the one-update case of a vocabulary and lambda"""
    B = 300 if (vname == "rico25" and lam == 3e6) else 40
    return B, B + VOCABS[vname].n_bins + int(lam) % 7


def multi_update_batch(vo: O.VocabSpec, n_up: int, centers: Optional[torch.Tensor], B: int = 40):
    """the several-update cases: at most 8 elements per layout.  After a large first update the boxes sit on bin centres,
    where touching boxes put edges exactly on a kink (linear centres especially); fewer edges per layout keep >= 90 % of
    the layouts well conditioned"""
    return make_batch(vo, B, 100 + n_up + vo.n_bins, centers, edge_p=0.22, n_max=8)


def centers_for(kind: str, n_bins: int) -> Optional[torch.Tensor]:
    """"none": no centres passed (the kernel's linear ones), "linear": float32(linspace) passed, "kmeans": non-uniform"""
    return {"none": None, "linear": linear_centers32(n_bins), "kmeans": kmeans_like_centers(n_bins, seed=n_bins)}[kind]


def kmeans_like_centers(n_bins: int, seed: int) -> torch.Tensor:
    """sorted, non-uniform centres in (0, 1] like a k-means fit: (4, n_bins) float32"""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for a in range(4):
        gaps = 0.3 + torch.rand(n_bins, generator=g, dtype=torch.float64) ** 2 * 2.0
        c = gaps.cumsum(0) / (gaps.sum() + 0.5 * gaps[0])
        rows.append(c if a >= 2 else c - c[0] * 0.9)
    return torch.stack(rows).float()


def make_batch(vo: O.VocabSpec, B: int, seed: int, centers: Optional[torch.Tensor], edge_p: float = 0.35, n_max: Optional[int] = None):
    """a relation batch with designed boxes.  Each element gets a target box; its bin logits peak at the target with a moderate
    spread (so p (c - b) is not 0) and the bbox tokens of x_t are MASK (a few are set), so the posterior keeps that shape.
    Layouts b % 8 == 3 have no edge (the kernel's early return), b % 8 == 5 hold a single element, b % 8 in (1, 6) also carry
    edges to and from PAD slots, which must be ignored.  -> cond (seq, mask, type, rel_adj), x_t, logits"""
    g = torch.Generator().manual_seed(seed)
    E, A, nb, nc = vo.n_elem, vo.n_attr, vo.n_bins, vo.n_cat
    cen = (linear_centers32(nb) if centers is None else centers).double()
    n_el = torch.randint(2, (n_max or E) + 1, (B,), generator=g)
    n_el[0] = n_max or E
    n_el[5::8] = 1
    seq = torch.full((B, vo.S), vo.mask_id, dtype=torch.long)
    mask = torch.zeros(B, vo.S, dtype=torch.bool)
    adj = torch.zeros(B, E + 1, E + 1, dtype=torch.int32)
    logits = torch.randn(B, vo.S, vo.C, generator=g) * 2.0
    x_t = torch.full((B, vo.S), vo.mask_id, dtype=torch.long)
    for b in range(B):
        n = int(n_el[b])
        seq[b, 0:A * n:A] = torch.randint(0, nc, (n,), generator=g)
        mask[b, 0:A * n:A] = True
        seq[b, A * n:] = vo.pad_id
        mask[b, A * n:] = True
        for e in range(n):
            tgt = torch.rand(4, generator=g, dtype=torch.float64) * (cen[:, -1] - cen[:, 0]) + cen[:, 0]
            sig = (0.02 + 0.05 * torch.rand(4, generator=g, dtype=torch.float64))[:, None]
            prof = -0.5 * ((cen - tgt[:, None]) / sig) ** 2 + 0.3 * torch.randn(4, nb, generator=g, dtype=torch.float64)
            for a in range(4):
                logits[b, A * e + 1 + a, nc + a * nb: nc + (a + 1) * nb] = (prof[a] + 6.0).float()
                if torch.rand(1, generator=g) < 0.08:
                    x_t[b, A * e + 1 + a] = nc + a * nb + int(torch.randint(0, nb, (1,), generator=g))
        if b % 8 == 3:
            continue
        for i in range(n + 1):
            for j in range(i + 1, n + 1):
                if torch.rand(1, generator=g) >= edge_p and not (n == 1 and i == 0):
                    continue
                size = int(torch.randint(0, 4, (1,), generator=g))
                if i == 0:
                    loc = [LOC_T, LOC_C, LOC_B, 4][int(torch.randint(0, 4, (1,), generator=g))]
                else:
                    loc = int(torch.randint(4, 10, (1,), generator=g))
                m = (1 << size) | (1 << loc)
                if m != (1 << 0 | 1 << 4):
                    adj[b, i, j] = m
        if b % 8 in (1, 6) and n < E:
            for _ in range(4):
                i = int(torch.randint(0, n + 1, (1,), generator=g))
                j = int(torch.randint(n + 1, E + 1, (1,), generator=g))
                m = (1 << int(torch.randint(1, 4, (1,), generator=g))) | (1 << int(torch.randint(5, 10, (1,), generator=g)))
                adj[b, i, j] = m
                adj[b, j, i] = m
    x_t = torch.where(mask, seq, x_t)
    return dict(seq=seq, mask=mask, type="relation", rel_adj=adj), x_t, logits


def posterior_input(vo: O.VocabSpec, x_t, logits, cond, t: int, T: int = 100) -> torch.Tensor:
    """the log-probs the update starts from (strong mask, no PAD-disable), fp32 oracle arithmetic: the CPU stand-in for the
    kernel's own input"""
    lx0 = O.predict_start(logits)
    lp = O.q_posterior(lx0, x_t, t, T, vo, O.group_schedules(T, vo, "constrained"), "constrained")
    strong = O.index_to_log_onehot(cond["seq"], vo.C)
    return torch.where(cond["mask"][..., None], strong, lp)
