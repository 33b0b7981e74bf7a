"""The side-feature layout every engine shares: which column block holds which modality, which feature table and Linear layer feed
it, and the order in which the fusion, the loss heads and the projection launches list the blocks.

Blocks (S = 2 + #attribute keys, d columns each) of Pi / Fu / Fi and their gradients:  img | txt | att_0 .. att_{S-3}.  Index S
stands for the user profile (the user table, user_trans, P_usr / prof_*).  Every list below keeps the order the reference
evaluates its terms in, and the order fixes bits: the fusion sums its terms in list order, the heads share Gprof_u in head order,
the grouped projections run their problems in list order, and the --drop_rate masks are drawn in the fusion list's order.
"""
from __future__ import annotations


class SideLayout:
    def __init__(self, keys, d):
        self.keys, self.d = list(keys), int(d)
        self.S = 2 + len(self.keys)
        # parameter prefix of block s, and of the user profile at index S (Models.py:145-150)
        self.weights = ["image_trans", "text_trans"] + ["item_trans"] * len(self.keys) + ["user_trans"]
        self.reg_weights = tuple(self.weights[:2])          # the layers of the feat_reg blocks (`reg`)

    def blk(self, buf, s):
        return buf[:, s * self.d:(s + 1) * self.d]

    def att(self, buf):
        """The attribute blocks of `buf`, in key order."""
        return [self.blk(buf, 2 + j) for j in range(len(self.keys))]

    def item_tables(self, f):
        """The feature tables of the S blocks (f: dict(image, text, item={key: table}, ...))."""
        return [f["image"], f["text"]] + [f["item"][k] for k in self.keys]

    def tables(self, f):
        """The feature tables of indices 0..S: the S blocks, then the user profile table."""
        return self.item_tables(f) + [f["user"]]

    def param(self, p, j):
        """(weight, bias) of index j from a dict keyed by parameter name (the parameters or their gradients)."""
        return p[self.weights[j] + ".weight"], p[self.weights[j] + ".bias"]

    # ---- the fusion (Models.py:185-197) -------------------------------------------------------------------------------------
    def fused(self, F, prof):
        """The side terms of one side's fusion: img, txt, profile, attributes (F: a column-block buffer, prof: the profile rows)."""
        return [self.blk(F, 0), self.blk(F, 1), prof] + self.att(F)

    def coefs(self, cfg):
        """The fusion weights of the `fused` terms."""
        return [cfg.model_cat_rate, cfg.model_cat_rate, cfg.user_cat_rate] + [cfg.item_cat_rate] * len(self.keys)

    # ---- the loss heads (main.py:238-254) --------------------------------------------------------------------------------------
    def heads(self, cfg, Fu, prof_u, GFu, Gprof_u, Fi, GFi):
        """The side-feature BPR heads that follow the ID head: image and text (user blocks 0 and 1 of Fu against the item blocks), then
        one head per attribute (the user profile against the attribute block).  Fu / GFu: any buffers whose blocks 0 and 1 hold the
        batch users' image and text rows and their gradients; prof_u / Gprof_u: the profile rows and their gradient."""
        b = self.blk
        return [(b(Fu, 0), b(Fi, 0), b(GFu, 0), b(GFi, 0), cfg.mm_mf_rate, 0.0),
                (b(Fu, 1), b(Fi, 1), b(GFu, 1), b(GFi, 1), cfg.mm_mf_rate, 0.0)] + \
               [(prof_u, x, Gprof_u, g, cfg.aug_mf_rate, 0.0) for x, g in zip(self.att(Fi), self.att(GFi))]

    # ---- feat_reg (main.py:151-156) -------------------------------------------------------------------------------------------
    def reg(self, F):
        """The blocks feat_reg covers: image and text, the first two (their layers: `reg_weights`)."""
        return F[:, :2 * self.d]

    def unreg(self, F):
        """The blocks feat_reg does not cover (the attributes)."""
        return F[:, 2 * self.d:]

    # ---- the grouped projection launches ---------------------------------------------------------------------------------------
    def proj_problems(self, f, p, Pi=None, P_usr=None, rows=None):
        """Problems of ops.proj_fwd_group (Models.py:145-150): each item-side table of f into its block of Pi (when given; rows: an
        optional row map of the tables into Pi), then the user table into P_usr (when given); long-K problems first, stably."""
        probs = []
        if Pi is not None:
            r = () if rows is None else (rows,)
            probs += [(X, *self.param(p, s), self.blk(Pi, s), *r) for s, X in enumerate(self.item_tables(f))]
        if P_usr is not None:
            probs.append((f["user"], *self.param(p, self.S), P_usr))
        probs.sort(key=lambda t: -t[0].shape[1])
        return probs

    def wgrad_problems(self, f, g, GPi, GP_usr, rows=None):
        """Problems of ops.proj_wgrad_group: the attribute blocks (one dW, accumulated after the first), the user profile, text, image
        -- the order in which item_trans's row chunks are summed.  g: the gradients by parameter name; rows: as in `proj_problems`."""
        r = () if rows is None else (rows,)
        X = self.item_tables(f)
        probs = [(X[s], self.blk(GPi, s), *self.param(g, s), s > 2, *r) for s in range(2, self.S)]
        probs.append((f["user"], GP_usr, *self.param(g, self.S), False))
        probs += [(X[s], self.blk(GPi, s), *self.param(g, s), False, *r) for s in (1, 0)]
        return probs
