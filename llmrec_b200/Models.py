"""MM_Model with the reference's constructor, parameter names and forward signature
(Models.py:19-199), executing on the sm_90a kernels of llmrec_b200.

Drop-in facts kept: parameter construction order (so a seeded CPU generator yields the reference's
initial weights, Models.py:30-42), state-dict names image_trans/text_trans/user_trans/item_trans/
user_id_embedding/item_id_embedding (+ the unused batch_norm), and the 14-tuple returned by
forward (Models.py:199).  The four image_/text_ graph arguments are accepted and ignored, as in the
reference.  Autograd works through one torch.autograd.Function whose backward is the hand-written
backward schedule of engine.HotPath.  The optional feature-mask / dropout / attribute-restoration branch (Models.py:131-142,203-225; main.py:258-271; off by default) is
the eager path of main.Trainer (`Trainer._train_batch_masked`, SURVEY.md 8f-4); the autograd entry point MM_Model.forward itself
raises for those flags instead of silently differing.
"""
import torch
import torch.nn as nn

from . import feat_int8
from .engine import HotPath, HotPathConfig, PARAM_ORDER
from .graph import operators_from_coo
from .ops import PROJ_MODE
from .runtime import get_args


class _HotPathFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hp, *params):
        hp.forward()
        hp._version = getattr(hp, "_version", 0) + 1
        ctx.hp, ctx.version = hp, hp._version
        return tuple(o.clone() for o, _ in hp.outputs())

    @staticmethod
    def backward(ctx, *g):
        hp = ctx.hp
        if ctx.version != hp._version:
            raise RuntimeError("MM_Model.forward was called again before backward; the fused path keeps one live forward")
        direct = None
        for (_, dst), src in zip(hp.outputs(), g):
            if dst is None:                                       # p_usr: its gradient is added in the backward chain
                direct = src.contiguous() if src is not None else None
            elif src is None:
                dst.zero_()
            else:
                dst.copy_(src)
        grads = hp.backward(gp_usr_direct=direct)
        return (None,) + tuple(grads[n].clone() for n in PARAM_ORDER)


def _on_device(t):
    """The kernels take device pointers: parameters must live on the GPU (the orchestration tests substitute this check together
    with the kernels, tests/ops_emulator.py)."""
    return t.is_cuda


class MM_Model(nn.Module):
    def __init__(self, n_users, n_items, embedding_dim, weight_size, dropout_list, image_feats, text_feats,
                 user_init_embedding, item_attribute_dict):
        super().__init__()
        args = get_args()
        self.n_users, self.n_items, self.embedding_dim = n_users, n_items, embedding_dim
        self.n_ui_layers = len(weight_size)
        self.weight_size = [embedding_dim] + list(weight_size)
        d = args.embed_size
        first = "title" if "title" in item_attribute_dict else next(iter(item_attribute_dict))
        # construction order == RNG order of the reference (Models.py:30-42)
        self.image_trans = nn.Linear(image_feats.shape[1], d)
        self.text_trans = nn.Linear(text_feats.shape[1], d)
        self.user_trans = nn.Linear(user_init_embedding.shape[1], d)
        self.item_trans = nn.Linear(item_attribute_dict[first].shape[1], d)
        for lin in (self.image_trans, self.text_trans, self.user_trans, self.item_trans):
            nn.init.xavier_uniform_(lin.weight)
        self.user_id_embedding = nn.Embedding(n_users, embedding_dim)
        self.item_id_embedding = nn.Embedding(n_items, embedding_dim)
        nn.init.xavier_uniform_(self.user_id_embedding.weight)
        nn.init.xavier_uniform_(self.item_id_embedding.weight)
        # --feat_dtype bf16: the constant feature tables are rounded once (torch's round-to-nearest-even cast; no RNG is drawn, so the
        # seeded parameter init above is unchanged) and stay bf16; the projection kernels read them as they are.  --feat_dtype int8:
        # quantized once into the row-scaled int8 format of feat_int8 (no RNG either); the kernels expand it to bf16 on chip
        feat_dtype = getattr(args, "feat_dtype", "fp32")
        if feat_dtype == "int8":
            as_feat = lambda a: feat_int8.quantize(torch.as_tensor(a).float()).contiguous()
        else:
            dt = torch.bfloat16 if feat_dtype == "bf16" else torch.float32
            as_feat = lambda a: torch.as_tensor(a).float().to(dt).contiguous()
        self.register_buffer("image_feats", as_feat(image_feats), persistent=False)
        self.register_buffer("text_feats", as_feat(text_feats), persistent=False)
        self.register_buffer("user_feats", as_feat(user_init_embedding), persistent=False)
        self._item_keys = list(item_attribute_dict.keys())
        for k in self._item_keys:
            self.register_buffer("item_feat__" + k, as_feat(item_attribute_dict[k]), persistent=False)
        self.batch_norm = nn.BatchNorm1d(d)      # present (unused) in the reference; kept for state_dict parity
        self.tau = 0.5
        self._hp = None
        self._hp_key = None

    @property
    def item_feats(self):
        return {k: getattr(self, "item_feat__" + k) for k in self._item_keys}

    def hot_path(self, ui_graph, iu_graph, hoisted=False, graph_scalars=None) -> HotPath:
        """The fused executor bound to this model's parameters and a (ui, iu) graph pair.  hoisted=True builds the engine of
        hoist.py (constant side-feature propagation precomputed; needs `graph_scalars` = BipartiteGraph.ones_propagated())."""
        key = (id(ui_graph), id(iu_graph), self.user_id_embedding.weight.data_ptr(), bool(hoisted))
        if self._hp is None or self._hp_key != key:
            args = get_args()
            if not _on_device(self.user_id_embedding.weight):
                raise RuntimeError("MM_Model runs on the H100 kernels only: move it to CUDA first (no CPU path)")
            ui_f, ui_b = operators_from_coo(ui_graph)
            iu_f, iu_b = operators_from_coo(iu_graph)
            params = {n: p.data for n, p in self.named_parameters() if n in PARAM_ORDER}
            feats = dict(image=self.image_feats, text=self.text_feats, user=self.user_feats, item=self.item_feats)
            cfg = HotPathConfig(embed_size=self.embedding_dim, n_layers=self.n_ui_layers, model_cat_rate=args.model_cat_rate,
                                user_cat_rate=args.user_cat_rate, item_cat_rate=args.item_cat_rate, aug_mf_rate=args.aug_mf_rate,
                                mm_mf_rate=args.mm_mf_rate, prune_loss_drop_rate=args.prune_loss_drop_rate,
                                feat_reg_decay=args.feat_reg_decay, regs0=eval(args.regs)[0], batch_size=args.batch_size,
                                aug_sample_rate=args.aug_sample_rate,
                                proj_mode=PROJ_MODE[getattr(args, "proj_mode", "3xtf32")],
                                deterministic=bool(getattr(args, "deterministic", 0)))
            if hoisted:
                from .hoist import HoistedHotPath
                self._hp = HoistedHotPath((ui_f, iu_f, ui_b, iu_b), params, feats, cfg, graph_scalars)
            else:
                self._hp = HotPath((ui_f, iu_f, ui_b, iu_b), params, feats, cfg)
            self._hp_key = key
        return self._hp

    def forward(self, ui_graph, iu_graph, image_ui_graph=None, image_iu_graph=None, text_ui_graph=None, text_iu_graph=None):
        args = get_args()
        if args.mask or args.mask_rate > 0 or args.drop_rate > 0:
            raise NotImplementedError("MM_Model.forward under autograd covers the default flags; the mask / dropout branch (Models.py:131-142) "
                                      "runs through main.Trainer (Trainer._train_batch_masked)")
        if args.layers < 1:
            raise NameError("args.layers must be >= 1 (the reference leaves image_user_feats undefined otherwise, Models.py:152)")
        hp = self.hot_path(ui_graph, iu_graph)
        params = [dict(self.named_parameters())[n] for n in PARAM_ORDER]
        out = _HotPathFn.apply(hp, *params)
        K = len(hp.keys)
        U, I, img_i, txt_i, img_u, txt_u, p_usr, prof_u, prof_i = out[:9]
        att_u = {k: out[9 + j] for j, k in enumerate(hp.keys)}
        att_i = {k: out[9 + K + j] for j, k in enumerate(hp.keys)}
        u_mask_nodes = torch.empty(0, dtype=torch.int64)          # int(mask_rate * n_users) == 0 (Models.py:139-141)
        return U, I, img_i, txt_i, img_u, txt_u, p_usr, att_i, prof_u, prof_i, att_u, att_i, None, u_mask_nodes


class Decoder(nn.Module):
    """Attribute-restoration head of the mask branch (Models.py:203-225): one Linear(embed_size -> feat_size) + LeakyReLU per side.
    The reference writes nn.LeakyReLU(True), i.e. negative_slope = 1.0 -- an identity; kept.  Constructed right after MM_Model so that
    the CPU generator is consumed in the reference's order (main.py:95-97); its optimizer is never stepped upstream (main.py:106-110)."""

    def __init__(self, feat_size):
        super().__init__()
        d = get_args().embed_size
        self.feat_size = feat_size
        self.u_net = nn.Sequential(nn.Linear(d, int(feat_size)), nn.LeakyReLU(True))
        self.i_net = nn.Sequential(nn.Linear(d, int(feat_size)), nn.LeakyReLU(True))

    def forward(self, u, i):
        """u: [n_u x d]; i: {key: [n_i x d]} -> ([n_u x feat], [n_keys x n_i x feat])"""
        return self.u_net(u.float()), self.i_net(torch.stack([i[k] for k in i.keys()]).float())
