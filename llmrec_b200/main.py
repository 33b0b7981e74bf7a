"""Trainer / CLI with the reference's interface (main.py:37-369) on the H100 hot path.

    python main.py --dataset netflix [all flags of utility/parser.py]

Kept: Trainer(data_config), .train(), .test(users, is_val), bpr_loss / prune_loss /
feat_reg_loss_calculation / csr_norm / matrix_to_tensor, the epoch log lines, NaN exit, early stopping.
Changed on purpose (same results, fewer host round trips):
  * the whole step (forward, 8 BPR heads + prune, backward, AdamW) is engine.HotPath.train_step;
    no per-head D2H argsort (main.py:159), no float(loss) syncs per step (:280-283) -- losses are
    accumulated on the device and read once per epoch;
  * augmented_sample_dict is unpickled once, not every batch (main.py:216; the file never changes);
  * the derived `*_final` / `augmented_total_embed_dict` files are NOT written back into the data
    directory (main.py:66,78 side effects);
  * clip_grad_norm_ before zero_grad (main.py:274) is a no-op upstream and is omitted.
Added (no counterpart upstream): checkpoints -- Trainer.save_checkpoint / load_checkpoint, --save_dir / --save_every / --resume /
--eval_only (checkpoint.py); without those flags nothing is written and train() is what it was.
"""
from __future__ import annotations

import math
import os
import pickle
import random
import sys
from datetime import datetime
from time import time

import numpy as np
import scipy.sparse as sp
import torch

from . import checkpoint, ops, recommend
from .Models import Decoder, MM_Model
from .graph import BipartiteGraph, histories_csr
from .runtime import get_args, set_args
from .utility import batch_test
from .utility.load_data import Data
from .utility.logging import Logger
from .utility.parser import parse_args, resolve_dataset_dir


def set_seed(seed):
    """main.py:355-359"""
    np.random.seed(seed)
    random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


class _StagingSlot:
    """One pinned [4 x cap] int32 index buffer (rows users / pos / neg / meta = {B', n_keep}) + the event recorded after its
    H2D copy.  A slot is rewritten only after that copy has completed, so the host may run ahead of the device by at most the
    ring length."""

    def __init__(self, cap):
        self.host = torch.zeros((4, cap), dtype=torch.int32).pin_memory()
        self.np = self.host.numpy()
        self.event = torch.cuda.Event()


def _stack_rows(obj):
    """indexable[n] -> ndarray [n x dim] (main.py:61-65, 73-77)."""
    if isinstance(obj, np.ndarray):
        return obj
    return np.array([obj[i] for i in range(len(obj))])


class Trainer(object):
    def __init__(self, data_config=None, data_generator=None, device="cuda"):
        args = self.args = get_args()
        if not torch.cuda.is_available():
            raise RuntimeError("llmrec_b200.Trainer needs a CUDA (H100) device: there is no CPU fallback")
        feat_dtype = getattr(args, "feat_dtype", "fp32")
        if feat_dtype in ("bf16", "int8") and (args.mask or args.mask_rate > 0):
            raise ValueError(f"--feat_dtype {feat_dtype} cannot be combined with --mask / --mask_rate > 0: the mask branch overwrites rows of the "
                             "feature tables with fp32 column means in place (Trainer._mask_features); use --feat_dtype fp32")
        if getattr(args, "deterministic", 0) and (args.mask or args.mask_rate > 0 or args.drop_rate > 0):
            raise ValueError("--deterministic 1 cannot be combined with --mask / --mask_rate > 0 / --drop_rate > 0: that branch accumulates with "
                             "torch's index_add_ and runs the Decoder backward, whose summation orders are not fixed")
        if getattr(args, "eval_only", 0) and not getattr(args, "resume", None):
            raise ValueError("--eval_only 1 evaluates a saved model: give it one with --resume PATH")
        if (getattr(args, "resume", None) or getattr(args, "save_dir", None)) and (args.mask or args.mask_rate > 0 or args.drop_rate > 0):
            raise ValueError("--save_dir / --resume cannot be combined with --mask / --mask_rate > 0 / --drop_rate > 0: that branch overwrites rows "
                             "of the feature tables for good (Trainer._mask_features), so the tables are run state there and a checkpoint "
                             "does not hold them")
        self.device = torch.device(device)
        self.task_name = "%s_%s_%s" % (datetime.now().strftime("%Y-%m-%d %H:%M:%S"), args.dataset, args.cf_model)
        self.logger = Logger(filename=self.task_name, is_debug=args.debug)
        self.logger.logging("PID: %d" % os.getpid())
        self.logger.logging(str(args))
        self.mess_dropout = eval(args.mess_dropout)
        self.lr, self.emb_dim, self.batch_size = args.lr, args.embed_size, args.batch_size
        self.weight_size = eval(args.weight_size)
        self.n_layers = len(self.weight_size)
        self.regs = eval(args.regs)
        self.decay = self.regs[0]

        ddir = self.data_dir = resolve_dataset_dir(args.data_path, args.dataset)
        if data_generator is None:
            data_generator = batch_test.data_generator
        if data_generator is None:
            data_generator = Data(path=ddir, batch_size=args.batch_size, sampler=getattr(args, "host_sampler", "python"))
        self.data_generator = data_generator
        batch_test.init(data_generator, args)

        rd = lambda name: pickle.load(open(os.path.join(ddir, name), "rb"))
        self.image_feats = np.load(os.path.join(ddir, "image_feat.npy"))                     # main.py:54-55
        self.text_feats = np.load(os.path.join(ddir, "text_feat.npy"))
        self.image_feat_dim, self.text_feat_dim = self.image_feats.shape[-1], self.text_feats.shape[-1]
        if os.path.exists(os.path.join(ddir, "train_mat")):
            self.ui_graph_raw = rd("train_mat")                                              # :59
        else:                                                                                # CSR store (utility/csr_store.py): same matrix, no pickle
            rowptr, col = data_generator.csr("train")
            self.ui_graph_raw = sp.csr_matrix((np.ones(col.shape[0], dtype=np.float32), col, rowptr),
                                              shape=(data_generator.n_users, data_generator.n_items))
        self.user_init_embedding = _stack_rows(rd("augmented_user_init_embedding"))          # :61-67
        raw_att = rd("augmented_atttribute_embedding_dict")                                  # :69-79
        self.item_attribute_embedding = {k: _stack_rows(raw_att[k]) for k in raw_att}
        self.augmented_sample_dict = rd("augmented_sample_dict")                             # :216 (loaded once)

        self.n_users, self.n_items = self.ui_graph_raw.shape                                 # :84-85
        self.graph = BipartiteGraph(self.ui_graph_raw, self.device)
        self.ui_graph, self.iu_graph = self.graph.coo_tensors()                              # :88-91
        self.image_ui_graph = self.text_ui_graph = self.ui_graph                             # :92-93
        self.image_iu_graph = self.text_iu_graph = self.iu_graph

        self.model_mm = MM_Model(self.n_users, self.n_items, self.emb_dim, self.weight_size, self.mess_dropout, self.image_feats,
                                 self.text_feats, self.user_init_embedding, self.item_attribute_embedding)   # built on CPU: RNG parity
        self.model_mm = self.model_mm.to(self.device)
        # main.py:97: the Decoder is built right after the model (its two nn.Linear inits consume the CPU generator before the first
        # torch.randperm of the mask branch); its optimizer exists upstream but is never stepped (main.py:106-110)
        self.decoder = Decoder(self.user_init_embedding.shape[1]).to(self.device)
        self.masked_mode = bool(args.mask) or args.mask_rate > 0 or args.drop_rate > 0
        # --hoist_side 1 (SURVEY.md 8f-3): only sound while dropout is the identity and the mask branch is off
        self.hoisted = bool(getattr(args, "hoist_side", 0)) and not (args.mask or args.mask_rate > 0 or args.drop_rate > 0)
        if self.hoisted:
            self.hot = self.model_mm.hot_path(self.ui_graph, self.iu_graph, hoisted=True, graph_scalars=self.graph.ones_propagated())
        else:
            self.hot = self.model_mm.hot_path(self.ui_graph, self.iu_graph)
        # torch.optim.AdamW defaults: betas (0.9, 0.999), eps 1e-8, weight_decay 0.01 (main.py:100-104)
        self.optimizer = self.hot.set_optimizer(lr=self.lr)
        self._slots, self._slot_i, self._idx_dev = [], 0, None
        # whole batches (users, items, augmented edges) from one C call, same `random` / `np.random` streams (host_native.BatchSampler)
        self._batch_sampler = None
        if getattr(data_generator, "_sampler", "python") == "native":
            from .host_native import BatchSampler
            rowptr, col = data_generator.csr("train")
            aug_pos, aug_neg = BatchSampler.aug_tables(self.augmented_sample_dict, data_generator.n_users, self.n_items)
            self._batch_sampler = BatchSampler(data_generator.exist_users, rowptr, col, data_generator.n_items, data_generator.batch_size,
                                               aug_pos, aug_neg, aug_limit=self.n_items)
            self._batch_np = np.empty((3, 2 * data_generator.batch_size + 8), dtype=np.int32)
        self.use_graph = bool(getattr(args, "cuda_graph", 1))
        self._epoch_stats = torch.zeros(4, dtype=torch.float32, device=self.device)          # total, mf, emb, interactions (device-side sampler)
        # --device_sampler 1 (SURVEY.md 8f-1): batches are drawn ON the GPU into the engine's index buffer, in front of every step
        # --device_sampler 2: the same place, drawing the host sampler's exact batches from device copies of `random` / `np.random`
        self.device_sampler = None
        self.ref_sampler = getattr(args, "device_sampler", 0) == 2 and not self.masked_mode
        if self.ref_sampler:
            from .device_sampler import ReferenceDeviceSampler
            from .host_native import BatchSampler
            rowptr, col = data_generator.csr("train")
            col_sorted = data_generator.csr("train", sorted_rows=True)[1]
            aug_pos, aug_neg = BatchSampler.aug_tables(self.augmented_sample_dict, data_generator.n_users, self.n_items)
            ds = self.device_sampler = ReferenceDeviceSampler(data_generator.exist_users, rowptr, col, col_sorted, data_generator.n_items,
                                                              data_generator.batch_size, aug_pos, aug_neg, self.n_items, args.aug_sample_rate,
                                                              self.device)
            # batch t + 1 is drawn beside step t (on the step's own stream with LLMREC_BRANCHES=0); the graph warm-up hands its batch back
            ds.attach(self.hot.index_buffer(self.hot.batch_capacity()), self.hot._meta_table, side_stream=self.hot.branches)
            self.hot.pre_step, self.hot.post_step = ds.step_begin, ds.step_end
            self.hot.pre_step_save, self.hot.pre_step_undo = ds.save, ds.undo
        elif getattr(args, "device_sampler", 0) and not self.masked_mode:
            from .device_sampler import DeviceSampler
            from .host_native import BatchSampler
            rowptr, col = data_generator.csr("train", sorted_rows=True)
            aug_pos, aug_neg = BatchSampler.aug_tables(self.augmented_sample_dict, data_generator.n_users, self.n_items)
            self.device_sampler = DeviceSampler(data_generator.exist_users, rowptr, col, data_generator.n_items, data_generator.batch_size,
                                                aug_pos, aug_neg, self.n_items, args.aug_sample_rate, self.device, seed=args.seed)
            gi = self.hot.index_buffer(self.hot.batch_capacity())
            self.hot.pre_step = lambda: self.device_sampler.fill(self.hot._gidx, self.hot._meta_table)
            self.hot.pre_step_undo = lambda: self.device_sampler.state[1:2].sub_(1)
        self.n_interactions = 0
        self._loop = self._new_loop()                 # where train() stands (what a checkpoint's `loop` section holds)
        self._resume_loop = None                      # set by load_checkpoint: the next train() continues from it
        # --resume: after set_seed and after the model and the Decoder were built, so their draws from the CPU generator happen as in
        # every run and the load then overwrites all RNG streams with the saved ones
        if getattr(args, "resume", None):
            self.load_checkpoint(args.resume)

    # ---- reference helper API (same names / returns) ----------------------------------------------
    def csr_norm(self, csr_mat, mean_flag=False):
        """main.py:114-126"""
        rowsum = np.array(csr_mat.sum(1))
        rowsum = np.power(rowsum + 1e-8, -0.5).flatten()
        rowsum[np.isinf(rowsum)] = 0.0
        left = sp.diags(rowsum) * csr_mat
        if mean_flag:
            return left
        colsum = np.array(csr_mat.sum(0))
        colsum = np.power(colsum + 1e-8, -0.5).flatten()
        colsum[np.isinf(colsum)] = 0.0
        return left * sp.diags(colsum)

    def matrix_to_tensor(self, cur_matrix):
        """main.py:128-134"""
        coo = cur_matrix.tocoo()
        idx = torch.from_numpy(np.vstack((coo.row, coo.col)).astype(np.int64))
        return torch.sparse_coo_tensor(idx, torch.from_numpy(coo.data), coo.shape).to(torch.float32).to(self.device)

    def prune_loss(self, pred, drop_rate):
        """Mean of the int((1-drop_rate)*n) smallest entries (main.py:158-165), selected on the device."""
        n_keep = int((1 - drop_rate) * len(pred))
        order = torch.argsort(pred.detach(), stable=True)
        return pred[order[:n_keep]].mean()

    def bpr_loss(self, users, pos_items, neg_items):
        """(mf_loss, emb_loss, reg_loss) of main.py:330-342 for pre-gathered rows (torch autograd API)."""
        pos_scores = torch.sum(users * pos_items, dim=1)
        neg_scores = torch.sum(users * neg_items, dim=1)
        regularizer = 1.0 / (2 * (users ** 2).sum() + 1e-8) + 1.0 / (2 * (pos_items ** 2).sum() + 1e-8) + 1.0 / (2 * (neg_items ** 2).sum() + 1e-8)
        regularizer = regularizer / self.batch_size
        maxi = torch.nn.functional.logsigmoid(pos_scores - neg_scores + 1e-8)
        mf_loss = -self.prune_loss(maxi, self.args.prune_loss_drop_rate)
        return mf_loss, self.decay * regularizer, 0.0

    def feat_reg_loss_calculation(self, g_item_image, g_item_text, g_user_image, g_user_text):
        """main.py:151-156"""
        feat_reg = 0.5 * (g_item_image ** 2).sum() + 0.5 * (g_item_text ** 2).sum() + 0.5 * (g_user_image ** 2).sum() + 0.5 * (g_user_text ** 2).sum()
        return self.args.feat_reg_decay * (feat_reg / self.n_items)

    # ---- evaluation ----------------------------------------------------------------------------------
    def test(self, users_to_test, is_val):
        """main.py:182-187: full forward in eval mode, then test_torch."""
        self.model_mm.eval()
        with torch.no_grad():
            if self.masked_mode:
                self._mask_features()                 # Models.py:131-142 runs in eval mode too (and keeps mutating the feature buffers)
            ua_embeddings, ia_embeddings = self.hot.forward()
        return batch_test.test_torch(ua_embeddings, ia_embeddings, users_to_test, is_val)

    # ---- optional branch: feature mask / dropout / attribute restoration (Models.py:131-150, main.py:258-271; SURVEY.md 8f-4) ---------
    def _mask_features(self):
        """Models.py:131-142: random rows of the attribute / profile tables are overwritten IN PLACE (persistently) with the column mean.
        torch.randperm draws from the CPU generator in the reference's order: items first (only with --mask), then users (always)."""
        args, m = self.args, self.model_mm
        i_mask = None
        if args.mask:
            i_mask = torch.randperm(self.n_items)[:int(args.mask_rate * self.n_items)].to(self.device)
            for k in m._item_keys:
                f = getattr(m, "item_feat__" + k)
                f[i_mask] = f.mean(0)
            self.hot.refresh_item_feats(i_mask)                           # the compact tables of the live items (engine.HotPath)
        u_mask = torch.randperm(self.n_users)[:int(args.mask_rate * self.n_users)].to(self.device)
        if u_mask.numel():                # (--drop_rate alone masks no row; a bf16 / int8 table has no fp32 mean to write)
            m.user_feats[u_mask] = m.user_feats.mean(0)
        return i_mask, u_mask

    @staticmethod
    def sce_criterion(x, y, alpha=1):
        """main.py:175-180"""
        x = torch.nn.functional.normalize(x, p=2, dim=-1)
        y = torch.nn.functional.normalize(y, p=2, dim=-1)
        return (1 - (x * y).sum(dim=-1)).pow(alpha).mean()

    @staticmethod
    def mse_criterion(x, y, alpha=3):
        """main.py:167-173 (the cosine term is computed and discarded upstream; the result is the MSE of the normalised rows)"""
        x = torch.nn.functional.normalize(x, p=2, dim=-1)
        y = torch.nn.functional.normalize(y, p=2, dim=-1)
        return torch.nn.functional.mse_loss(x, y)

    def _train_batch_masked(self, u, p, n):
        """One training step with --mask / --mask_rate / --drop_rate: the same kernels, launched eagerly, with the branch-specific pieces
        (feature masking, dropout masks, Decoder + restoration loss) as plain torch ops between them.  Off by default upstream."""
        args, hp, m = self.args, self.hot, self.model_mm
        i_mask, u_mask = self._mask_features()
        hp._proj_fwd()
        drop = None
        if args.drop_rate > 0:
            # nn.Dropout in training mode on each projection, reference order image, text, user, item keys (Models.py:145-150); the mask of a
            # contiguous [n x d] tensor is drawn from the CUDA generator exactly as nn.Dropout would on the projection itself
            blocks = hp.sides.fused(hp.Pi, hp.P_usr)
            drop = [torch.nn.functional.dropout(torch.ones(b.shape[0], hp.d, device=self.device), p=args.drop_rate, training=True) for b in blocks]
            for b, mk in zip(blocks, drop):
                b.mul_(mk)
        hp._prop_fwd()
        hp._fuse_fwd()
        hp.loss_and_output_grads(u, p, n)
        if args.mask and args.att_re_rate != 0:
            # main.py:258-271: decoder on the DETACHED masked profile rows (torch.tensor(...) upstream copies) and on the masked rows of the
            # propagated attribute features (these keep their graph: the gradient flows back into GFi)
            v = hp.side_views()
            keys = hp.keys
            leaf = {k: v["att_i"][k][i_mask].detach().clone().requires_grad_(True) for k in keys}
            dec_u, dec_i = self.decoder(v["prof_u"][u_mask].detach(), leaf)
            crit = self.mse_criterion if args.feat_loss_type == "mse" else self.sce_criterion
            raw_u = torch.as_tensor(self.user_init_embedding[u_mask.cpu().numpy()], device=self.device).float()
            att = crit(dec_u, raw_u, alpha=args.alpha_l)
            for j, k in enumerate(keys):
                raw_i = torch.as_tensor(self.item_attribute_embedding[k][i_mask.cpu().numpy()], device=self.device).float()
                att = att + crit(dec_i[j], raw_i, alpha=args.alpha_l)
            (args.att_re_rate * att).backward()
            self.decoder.zero_grad(set_to_none=True)                      # de_optimizer is never stepped upstream
            for k, g in hp.side_views(grads=True)["att_i"].items():
                g.index_add_(0, i_mask, leaf[k].grad)
            hp.loss.add_(args.att_re_rate * att.detach())
        hp._fuse_bwd()
        hp._chain_bwd()
        if drop is not None:                                              # backward of the dropout: the same masks on the projection gradients
            for b, mk in zip(hp.sides.fused(hp.GPi, hp.GP_usr), drop):
                b.mul_(mk)
        hp._wgrad()
        hp.opt.step([hp.grads[k] for k in hp._opt_names])
        self._last_dropout_masks = drop
        return hp.loss

    # ---- one batch ---------------------------------------------------------------------------------------
    def sample_batch(self):
        """Data.sample() + augmented edges (main.py:213-224); host side, reference RNG order.  -> three lists."""
        if self._batch_sampler is not None:
            o = self._batch_np
            B = self._batch_sampler.draw(o, self.args.aug_sample_rate)
            self.new_batch_size = B - self._batch_sampler.batch
            return o[0, :B].tolist(), o[1, :B].tolist(), o[2, :B].tolist()
        users, pos_items, neg_items = self.data_generator.sample()
        aug = self.augmented_sample_dict
        ni = self.n_items
        users_aug = random.sample(users, int(len(users) * self.args.aug_sample_rate))
        keep = [u for u in users_aug if (aug[u][0] < ni and aug[u][1] < ni)]
        self.new_batch_size = len(keep)
        users = users + keep
        # a negative augmented id passes upstream's filter and wraps under Python indexing (row -1 = last item): same row here
        pos_items = pos_items + [aug[u][0] % ni for u in keep]
        neg_items = neg_items + [aug[u][1] % ni for u in keep]
        return users, pos_items, neg_items

    def _next_slot(self, need):
        """Next pinned staging slot of the ring (4 slots), free to be rewritten.  The device side of the copy is the engine's
        static index buffer (what the captured CUDA graph reads), so a batch crosses PCIe exactly once."""
        self._idx_dev = self.hot.index_buffer(need)
        cap = self._idx_dev.shape[1]
        if not self._slots or self._slots[0].host.shape[1] != cap:
            if self._slots:
                torch.cuda.synchronize()                                  # copies out of the old ring may still be in flight
            self._slots = [_StagingSlot(cap) for _ in range(4)]
            self._slot_i = 0
        slot = self._slots[self._slot_i]
        self._slot_i = (self._slot_i + 1) % len(self._slots)
        slot.event.synchronize()                                          # its previous H2D copy has completed
        return slot

    def _push(self, slot, B):
        slot.np[3, 0:2] = self.hot.meta_row(B)                            # {B', n_keep}: the graph's kernels read them from the device
        w = max(B, 2)
        self._idx_dev[:, :w].copy_(slot.host[:, :w], non_blocking=True)
        slot.event.record()
        self.last_h2d_bytes = 4 * 4 * w
        d = self._idx_dev
        return d[0, :B], d[1, :B], d[2, :B]

    def upload_batch(self, users, pos_items, neg_items):
        """[3 x B'] int32 through pinned memory; returns three device views."""
        B = len(users)
        slot = self._next_slot(B)
        slot.np[0, :B] = users
        slot.np[1, :B] = pos_items
        slot.np[2, :B] = neg_items
        return self._push(slot, B)

    def stage_batch(self):
        """sample_batch + upload_batch without the Python lists in between: the C sampler writes the batch straight into
        a pinned staging slot.  -> three device views (users, pos, neg)."""
        if self._batch_sampler is None:
            return self.upload_batch(*self.sample_batch())
        slot = self._next_slot(self.hot.batch_capacity())
        B = self._batch_sampler.draw(slot.np[:3], self.args.aug_sample_rate)
        self.new_batch_size = B - self._batch_sampler.batch
        return self._push(slot, B)

    def _step(self, u, p, n):
        # u, p, n are views of the engine's index buffer (see _push): the graph replays on what was just staged
        if self.masked_mode:
            loss = self._train_batch_masked(u, p, n)
        else:
            loss = self.hot.replay_staged() if self.use_graph else self.hot.train_step(u, p, n)
        # device-side epoch accumulators: [total, mf(main), emb(main)]
        self._epoch_stats[0:1] += loss
        self._epoch_stats[1:3] += self.hot.head_out[0:2]
        return loss

    def train_batch(self, users, pos_items, neg_items):
        return self._step(*self.upload_batch(users, pos_items, neg_items))

    def train_next_batch(self):
        """One iteration of the training loop (main.py:213-278): draw the next batch, run the step.  -> (loss tensor, B').
        With the device-side sampler B' is only known on the device (-1 here; Trainer.train reads the epoch total once)."""
        if self.device_sampler is not None:
            hp = self.hot
            if self.ref_sampler:
                self.device_sampler.host_is_current = False
            if self.use_graph:
                loss = hp.replay_staged()
            else:
                hp.pre_step()
                gi = hp._gidx
                loss = hp.train_step(gi[0], gi[1], gi[2], gi[3])
                if hp.post_step is not None:
                    hp.post_step()
            self._epoch_stats[0:1] += loss
            self._epoch_stats[1:3] += hp.head_out[0:2]
            self._epoch_stats[3:4] += hp._gidx[3, 0:1].float()
            return loss, -1
        u, p, n = self.stage_batch()
        return self._step(u, p, n), int(u.numel())

    # ---- checkpoints (checkpoint.py: format, durable write, validated read) -------------------------------
    @staticmethod
    def _new_loop():
        return dict(epoch=0, batch=0, best_recall=0, stopping_step=0, test_ret=None)

    def _fingerprint(self):
        """must: what a checkpoint has to agree with to be loadable at all; recorded: the flags an exact resume needs equal."""
        args = self.args
        live = checkpoint.engine_tensors(self.hot)
        must = dict(n_users=int(self.n_users), n_items=int(self.n_items), train_nnz=int(self.ui_graph_raw.nnz), embed_size=int(self.emb_dim),
                    weight_size=tuple(int(w) for w in self.weight_size),
                    feat_widths=tuple(int(t.shape[1]) for t in (self.image_feats, self.text_feats, self.user_init_embedding,
                                                                 *self.item_attribute_embedding.values())),
                    params={k[len("model/"):]: tuple(t.shape) for k, t in live.items() if k.startswith("model/")})
        flags = ("seed", "batch_size", "lr", "regs", "model_cat_rate", "user_cat_rate", "item_cat_rate", "aug_mf_rate", "mm_mf_rate",
                 "prune_loss_drop_rate", "feat_reg_decay", "aug_sample_rate", "proj_mode", "feat_dtype", "hoist_side", "device_sampler",
                 "host_sampler", "deterministic", "cuda_graph")
        return dict(must=must, recorded={k: getattr(args, k) for k in flags})

    def save_checkpoint(self, path):
        """Write the whole run state to `path`, at a step boundary: parameters, AdamW moments and step block, the RNG streams the samplers
        advance, and where the training loop stands.  Synchronises once, for the device-to-host copies; a training step never does."""
        live = dict(checkpoint.engine_tensors(self.hot), epoch_stats=self._epoch_stats)
        if self.ref_sampler:
            self.device_sampler.sync_to_host()                        # the file holds `random` / `np.random` as a host-sampled run has them
        elif self.device_sampler is not None:
            live["device_sampler"] = self.device_sampler.state
        host = checkpoint.to_host(live)
        model, optim = checkpoint.engine_sections(host, self.hot.opt)
        lp = self._loop
        ret = lp["test_ret"]
        loop = dict(epoch=int(lp["epoch"]), batch=int(lp["batch"]), epoch_stats=host["epoch_stats"], best_recall=float(lp["best_recall"]),
                    stopping_step=int(lp["stopping_step"]), n_interactions=int(self.n_interactions),
                    test_ret=None if ret is None else {k: float(v) if np.ndim(v) == 0 else torch.as_tensor(np.asarray(v, dtype=np.float64))
                                                       for k, v in ret.items()})
        checkpoint.write(path, model, optim, checkpoint.rng_state(self.device, host.get("device_sampler")), loop, self._fingerprint())

    def load_checkpoint(self, path):
        """Put the state of `save_checkpoint` back, IN PLACE (HotPath.load_state): before the first step or after a CUDA graph has been
        captured and replayed.  The file is validated as a whole first; a load that raises leaves this Trainer as it was.  The next
        train() continues from the saved epoch and batch.  A recorded flag that differs from this run's is logged; the continuation is
        exact only when none does."""
        ck, saved, diffs = checkpoint.read(path, self._fingerprint(), checkpoint.engine_tensors(self.hot))
        if diffs:
            self.logger.logging("checkpoint %s was written with other flags (saved -> this run): %s" % (path, ", ".join(diffs)))
        self.hot.load_state(saved)
        checkpoint.set_rng_state(ck["rng"], self.device, None if self.ref_sampler else self.device_sampler)
        if self.ref_sampler:
            self.device_sampler.upload_from_host()                    # in place, also under a captured graph
        lp = ck["loop"]
        self._epoch_stats.copy_(lp["epoch_stats"])
        self.n_interactions = lp["n_interactions"]
        ret = lp["test_ret"]
        self._loop = self._resume_loop = dict(
            epoch=lp["epoch"], batch=lp["batch"], best_recall=lp["best_recall"], stopping_step=lp["stopping_step"],
            test_ret=None if ret is None else {k: v.numpy() if isinstance(v, torch.Tensor) else v for k, v in ret.items()})

    def evaluate(self):
        """--eval_only 1: no training step; the metrics of the loaded model on the test users, logged like an epoch's."""
        ret = self.test(list(self.data_generator.test_set.keys()), is_val=False)
        r, p, h, n = ret["recall"], ret["precision"], ret["hit_ratio"], ret["ndcg"]
        self.logger.logging("recall=[%.5f, %.5f, %.5f, %.5f], precision=[%.5f, %.5f, %.5f, %.5f], hit=[%.5f, %.5f, %.5f, %.5f], "
                            "ndcg=[%.5f, %.5f, %.5f, %.5f]" % (r[0], r[1], r[2], r[-1], p[0], p[1], p[2], p[-1], h[0], h[1], h[2], h[-1],
                                                               n[0], n[1], n[2], n[-1]))
        return ret

    # ---- recommendations (recommend.py) ---------------------------------------------------------------------------------
    def _current_model(self):
        """The engine after a full eval forward: a training step leaves U / I current on its batch's rows only, and every item-side
        tensor one parameter update behind.  Launches nothing else and changes no run state."""
        if self.masked_mode:
            raise ValueError("recommendations need a fixed model: with --mask / --mask_rate > 0 / --drop_rate > 0 every forward rewrites rows of "
                             "the feature tables (Trainer._mask_features)")
        recommend.check_engine(self.hot)
        with torch.no_grad():
            self.hot.forward()
        return self.hot

    def recommend(self, users=None, K=10, exclude="train", histories=None, new_items=None, among=None, exclude_items=None, diversity=None,
                  pool=None):
        """-> (ids int64 [m x K], scores fp32 [m x K]) on the device: each row's K best items, ties to the lowest item id, padded with
        -1 / -inf when fewer than K items are left.
        users: trained user ids (default every user).  histories: item-id lists or a (rowptr, col) pair, folded in with the trained item
        side (HotPath.fold_in); `users` then names each history's trained id (or -1) and may be omitted.  new_items: the user lists of m
        items added after training (user-id lists or a (rowptr, col) pair), folded in with the trained user side (HotPath.fold_in_items)
        and scored after the trained catalog as ids n_items + j.  exclude: "train" masks a trained user's training items and a history's
        own items, and every new item whose list names the user (a history: its trained id); "none" masks nothing (the reference's
        candidate lists).
        among: rank only these item ids (an int list, ndarray or tensor; ids in [0, n_items + m), so new item j is n_items + j; order
        and repeats do not matter); None ranks the whole catalog.  exclude_items: per query, item ids to leave out on top of `exclude`
        (one row per query: id lists, a (rowptr, col) pair, or a 2-D array [m x C] with -1 as padding; ids in [0, n_items + m)); it
        only hides items, the scores are unchanged.  Returned ids are catalog ids either way.
        K: 1..64, at most the catalog size and at most the number of distinct ids in `among`.
        diversity: None, or lambda in [0, 1] for a diversified list: the K items are picked greedily from the row's own top-`pool` list,
        first the best-scored, then each time the item with the largest lambda * score - (1 - lambda) * (its largest cosine to an item
        already picked), cosines those of `similar_items` (recommend.diversify); rows come back in pick order with their scores.
        lambda = 1 gives the first K of the pool.  pool: K..64, default the smallest of 64 and the number of rankable ids.
        Every argument is checked before anything runs.  --proj_mode picks the scoring mode."""
        job = recommend.prepare_top_k(self.hot, self.graph.rowptr_u, self.graph.col_u, users=users, K=K, exclude=exclude,
                                      histories=histories, new_items=new_items, among=among, exclude_items=exclude_items,
                                      diversity=diversity, pool=pool)
        hot = self._current_model()
        mode = ops.SCORE_MODE.get(getattr(self.args, "proj_mode", "3xtf32"), 0)
        return recommend.run_top_k(hot, job, mode)

    def recommend_groups(self, groups, K=10, agg="mean", exclude="train", new_items=None, among=None, exclude_items=None):
        """-> (ids int64 [g x K], scores fp32 [g x K]) on the device: one list per group of trained users who choose together, ties to
        the lowest item id, padded with -1 / -inf when fewer than K items are left.
        groups: user-id lists or a (rowptr, col) pair, one row per group; repeats collapse and order does not matter; 1..64 distinct
        members per group.  A group's score of an item, with s(u, i) the bits `score` returns: agg="mean" the fp32 sum of s(u, i) over
        the members in ascending id, then one division by their number; "min" the least misery, "max" the most pleasure (exact; a NaN
        member score makes the group's NaN).  An item whose group score is NaN or -inf is never returned.
        exclude: "train" masks every member's training items and every new item whose list names a member; "none" masks nothing.
        new_items / among: as for `recommend`.  exclude_items: per group, item ids to leave out on top of `exclude` (one row per group,
        in the forms `recommend` takes).  K: 1..64, at most the catalog size and at most the number of distinct ids in `among`.
        A group of one member [u] gets exactly `recommend(users=[u])`'s row, and a group's row does not depend on the other groups of
        the call -- in --proj_mode 3xtf32 unless group scores closer than the tensor-core rounding straddle the selection's slack (the
        slack follows the size of the call, as for `recommend`).  Every argument is checked before anything runs.  --proj_mode picks the
        scoring mode; both give the same ids and bits under the same proviso."""
        job = recommend.prepare_group_top_k(self.hot, self.graph.rowptr_u, self.graph.col_u, groups, K=K, agg=agg, exclude=exclude,
                                            new_items=new_items, among=among, exclude_items=exclude_items)
        hot = self._current_model()
        mode = ops.SCORE_MODE.get(getattr(self.args, "proj_mode", "3xtf32"), 0)
        return recommend.run_group_top_k(hot, job, mode)

    def fold_in(self, histories, known=None):
        """-> U_new [m x d]: the fused user representations of item-id histories (lists or a (rowptr, col) pair) under the current
        parameters; known: each history's trained user id or -1 (layer 0 = that user's ID embedding, or zero)."""
        R = histories_csr(histories, self.n_items)
        return self._current_model().fold_in(R.indptr, R.indices, known=known)

    def fold_in_items(self, user_lists, known=None):
        """-> I_new [m x d]: the fused item representations of items given by the trained users who interacted with each (user-id lists
        or a (rowptr, col) pair) under the current parameters; known: each item's trained id or -1 (layer 0 = that item's ID embedding,
        or zero).  No feature rows are needed: an item's own side features do not enter its row."""
        R = recommend.new_items_csr(user_lists, self.n_users)
        if R is None:
            raise ValueError("fold_in_items: give one user-id list per item")
        return self._current_model().fold_in_items(R.indptr, R.indices, known=known)

    def similar_items(self, items, K=10, new_items=None, among=None):
        """-> (ids int64 [q x K], cosines fp32 [q x K]) on the device: each query item's K nearest items by cosine of the fused item rows,
        never the query itself, ties to the lowest id, padded with -1 / -inf.  items: trained ids, or n_items + j for the j-th of
        `new_items` (user lists of items added after training, as for `recommend`).  among: the neighbours come only from these item
        ids (as for `recommend`; a query need not be one of them); None = the whole catalog.  K: 1..64 and below the catalog size, or
        with `among` at most its number of distinct ids."""
        Rn = recommend.new_items_csr(new_items, self.n_users)
        n = self.n_items + (0 if Rn is None else Rn.shape[0])
        if among is None:
            recommend.check_k(K, n - 1, "the catalog size - 1")
        else:
            recommend.check_k(K, recommend.catalog_ids(among, n, self.hot.E_u.device).numel(), "|among|")
        hot = self._current_model()
        mode = ops.SCORE_MODE.get(getattr(self.args, "proj_mode", "3xtf32"), 0)
        return recommend.similar_items(hot, items, K=K, new_items=Rn, mode=mode, among=among)

    def score(self, users, items, new_items=None):
        """-> fp32 [n] on the device: the model's score <U[users[p]], I[items[p]]> of each (user, item) pair, by the exact fp32 chain of the
        scores `recommend` returns (the same pair gets the same bits; --proj_mode does not change them).  users: trained ids; items:
        trained ids, or n_items + j for the j-th of `new_items` (user lists of items added after training, folded in as for `recommend`).
        Equal lengths; ids are checked before anything runs."""
        Rn = recommend.new_items_csr(new_items, self.n_users)
        u, i = recommend.check_pairs(users, items, self.n_users, self.n_items + (0 if Rn is None else Rn.shape[0]))
        return recommend.score_pairs(self._current_model(), u, i, new_items=Rn)

    def rerank(self, candidates, users=None, K=None, exclude="none", histories=None, new_items=None, diversity=None, pool=None):
        """-> (ids int64 [m x K], scores fp32 [m x K]) on the device: each query's candidate list ordered by this model, the K best by
        (score desc, id asc), padded with -1 / -inf.  candidates: a sequence of item-id lists, a (rowptr, col) pair, or a 2-D integer
        tensor / ndarray [m x C] (the `candidate_indices` layout; -1 = padding); ids in [0, n_items + len(new_items)).  Queries as in
        `recommend`: trained users (default every user, when there is one candidate row per user) or `histories` folded in, `users` then
        naming each history's trained id (or -1).  Repeated ids are kept once.  exclude: "none" (default: a given shortlist is not thinned)
        or "train" (drops what `recommend` masks).  K: 1..1024, None = the longest surviving row.  Scores are exact fp32 in every
        --proj_mode, bit-identical to `recommend`'s for the same (user, item).
        diversity / pool: a diversified list as for `recommend`, picked from each row's own re-ranked top-`pool` list; pool: K..1024,
        default the smallest of 1024 and the longest surviving row (at least K); K=None then means K = pool."""
        job = recommend.prepare_rerank(self.hot, self.graph.rowptr_u, self.graph.col_u, candidates, users=users, K=K, exclude=exclude,
                                       histories=histories, new_items=new_items, diversity=diversity, pool=pool)
        return recommend.run_rerank(self._current_model(), job)

    def explain(self, items, users=None, histories=None, new_items=None, top=None):
        """-> recommend.Explanation on the device: why this model scores each query's targets as it does.  Each score <U[u], I[i]> splits
        exactly into one term per (history item, channel) -- channels "id", "image", "text", "profile" and one per attribute key (only
        "id" without side features) -- plus `own` (the user's ID embedding) and `last` (the softmax layer l = L), which are not linear in
        the history.  items: each query's targets, in the forms `rerank` takes for candidates (`ids` from `recommend` goes straight in;
        -1 = padding, whose outputs are zeros).  Queries as in `recommend`: trained users (default every user, with one target row per
        user), whose history is their training row, or `histories` folded in, `users` then naming each history's trained id (or -1: no
        ID embedding, own = 0).  new_items: user lists of items added after training; target n_items + j is the j-th.  top: None, or N
        in 1..64 for each target's N history items with the largest summed contribution.  Every argument is checked before anything
        runs; the outputs are exact fp32, the same bits whatever else is in the call."""
        job = recommend.prepare_explain(self.hot, self.graph.rowptr_u, self.graph.col_u, items, users=users, histories=histories,
                                        new_items=new_items, top=top)
        return recommend.run_explain(self._current_model(), job)

    def write_rerank(self, path, candidates, K):
        """--rerank_out: every user's candidate row (`candidate_indices` layout [n_users x C]) re-ranked by this model, nothing excluded,
        top K, pickled as a CPU int64 tensor [n_users x K] to `path` (atomically, as `write_candidates`)."""
        ids, _ = self.rerank(candidates, K=K)
        return recommend.write_candidates(path, ids)

    def write_groups(self, path, groups, K=10, agg="mean"):
        """--groups_out: the top-K of every group of `groups` (--groups_in) under `agg`, each group's training items excluded, pickled
        as a CPU int64 tensor [n_groups x K] to `path` (atomically, as `write_candidates`)."""
        ids, _ = self.recommend_groups(groups, K=K, agg=agg, exclude="train")
        return recommend.write_candidates(path, ids)

    def write_candidates(self, path, K=10, among=None, diversity=None, pool=None):
        """--candidates_out: the top-K of every user over the whole catalog, or over the item ids `among` (--candidates_among), nothing
        excluded (torch.topk(U . I^T, k=K) of the reference's stage 1), or with `diversity` (--candidates_diversity, --candidates_pool) the
        diversified K of `recommend`, pickled as a CPU int64 tensor [n_users x K] to `path` (atomically)."""
        ids, _ = self.recommend(K=K, exclude="none", among=among, diversity=diversity, pool=pool)
        return recommend.write_candidates(path, ids)

    # ---- training loop (main.py:189-326) -----------------------------------------------------------------
    def train(self):
        """Starts at epoch 0, or where the checkpoint loaded last stands: in the middle of an epoch its remaining batches run on top of
        the saved loss accumulators, so the epoch's log line is the uninterrupted one, and early stopping keeps its counters."""
        args, dg = self.args, self.data_generator
        run_time = datetime.strftime(datetime.now(), "%Y_%m_%d__%H_%M_%S")
        training_time_list = []
        lp = self._loop = self._resume_loop or self._new_loop()
        self._resume_loop = None
        save_dir = getattr(args, "save_dir", None)
        save_every = max(int(getattr(args, "save_every", 1)), 1)
        stopping_step, best_recall, test_ret = lp["stopping_step"], lp["best_recall"], lp["test_ret"]
        if self.ref_sampler and self.device_sampler.host_is_current:
            self.device_sampler.upload_from_host()                    # from `random` / `np.random` as they stand now, like the host sampler
        for epoch in range(lp["epoch"], args.epoch):
            t1 = time()
            n_batch = dg.n_train // args.batch_size + 1
            if lp["batch"] == 0:
                self._epoch_stats.zero_()
                self.n_interactions = 0
            self.model_mm.train()
            for k in range(lp["batch"], n_batch):
                self.n_interactions += max(self.train_next_batch()[1], 0)
                lp["batch"] = k + 1
            loss, mf_loss, emb_loss, n_dev = (float(x) for x in self._epoch_stats.tolist())      # the one sync per epoch
            if self.ref_sampler:
                self.device_sampler.check()                           # a draw that failed on the device raises here
            self.n_interactions += int(n_dev)
            reg_loss, contrastive_loss = 0.0, 0.0
            if math.isnan(loss):
                self.logger.logging("ERROR: loss is nan.")
                sys.exit()
            if (epoch + 1) % args.verbose != 0:
                self.logger.logging("Epoch %d [%.1fs]: train==[%.5f=%.5f + %.5f + %.5f  + %.5f]" % (
                    epoch, time() - t1, loss, mf_loss, emb_loss, reg_loss, contrastive_loss))
                training_time_list.append(time() - t1)
            t2 = time()
            users_to_test = list(dg.test_set.keys())
            ret = self.test(users_to_test, is_val=False)
            training_time_list.append(t2 - t1)
            t3 = time()
            self.last_epoch_times = (t2 - t1, t3 - t2)
            if args.verbose > 0:
                r, p, h, n = ret["recall"], ret["precision"], ret["hit_ratio"], ret["ndcg"]
                self.logger.logging(
                    "Epoch %d [%.1fs + %.1fs]: train==[%.5f=%.5f + %.5f + %.5f], recall=[%.5f, %.5f, %.5f, %.5f], "
                    "precision=[%.5f, %.5f, %.5f, %.5f], hit=[%.5f, %.5f, %.5f, %.5f], ndcg=[%.5f, %.5f, %.5f, %.5f]" % (
                        epoch, t2 - t1, t3 - t2, loss, mf_loss, emb_loss, reg_loss, r[0], r[1], r[2], r[-1], p[0], p[1], p[2], p[-1],
                        h[0], h[1], h[2], h[-1], n[0], n[1], n[2], n[-1]))
            lp.update(epoch=epoch + 1, batch=0)                # a checkpoint written from here on continues with the next epoch
            if ret["recall"][1] > best_recall:
                best_recall = ret["recall"][1]
                test_ret = self.test(users_to_test, is_val=False)
                self.logger.logging("Test_Recall@%d: %.5f,  precision=[%.5f], ndcg=[%.5f]" % (
                    eval(args.Ks)[1], test_ret["recall"][1], test_ret["precision"][1], test_ret["ndcg"][1]))
                stopping_step = 0
                lp.update(best_recall=best_recall, test_ret=test_ret, stopping_step=0)
                if save_dir:
                    self.save_checkpoint(os.path.join(save_dir, "best.pt"))      # the parameters that scored it
            elif stopping_step < args.early_stopping_patience:
                stopping_step += 1
                lp["stopping_step"] = stopping_step
                self.logger.logging("#####Early stopping steps: %d #####" % stopping_step)
            else:
                self.logger.logging("#####Early stop! #####")
                break
            if save_dir and (epoch + 1) % save_every == 0:
                self.save_checkpoint(os.path.join(save_dir, "last.pt"))
        if self.ref_sampler:
            self.device_sampler.sync_to_host()                        # `random` / `np.random` end where a host-sampled run leaves them
        self.logger.logging(str(test_ret))
        return best_recall, run_time


def main(argv=None):
    args = set_args(parse_args(argv))
    os.environ.setdefault("CUDA_VISIBLE_DEVICES", str(args.gpu_id))
    set_seed(args.seed)
    ddir = resolve_dataset_dir(args.data_path, args.dataset)
    gen = Data(path=ddir, batch_size=args.batch_size, sampler=args.host_sampler)
    batch_test.init(gen, args)
    config = dict(n_users=gen.n_users, n_items=gen.n_items)
    cand_among = check_candidates_flags(args, gen.n_items)           # before any training: a bad K, file or flag mix fails at once
    trainer = Trainer(data_config=config, data_generator=gen)         # --resume loads here, after set_seed and the model's own draws
    if args.candidates_out and trainer.masked_mode:
        raise ValueError("--candidates_out needs a fixed model: not with --mask / --mask_rate > 0 / --drop_rate > 0")
    rerank_in, rerank_k = check_rerank_flags(args, trainer)
    groups_in = check_groups_flags(args, trainer)
    ret = trainer.evaluate() if args.eval_only else trainer.train()
    if args.candidates_out:                                           # from the model in memory when the run ends
        trainer.write_candidates(args.candidates_out, args.candidates_k, among=cand_among, diversity=args.candidates_diversity,
                                 pool=args.candidates_pool)
        trainer.logger.logging("candidates: top-%d of %d users written to %s" % (args.candidates_k, trainer.n_users, args.candidates_out))
    if rerank_in is not None:
        trainer.write_rerank(args.rerank_out, rerank_in, rerank_k)
        trainer.logger.logging("rerank: %d users' candidates from %s, top-%d written to %s" % (trainer.n_users, args.rerank_in, rerank_k,
                                                                                              args.rerank_out))
    if groups_in is not None:
        trainer.write_groups(args.groups_out, groups_in, args.groups_k, args.groups_agg)
        trainer.logger.logging("groups: top-%d (%s) of %d groups from %s written to %s" % (args.groups_k, args.groups_agg, groups_in[0].numel() - 1,
                                                                                           args.groups_in, args.groups_out))
    return ret


def check_candidates_flags(args, n_items):
    """--candidates_out / --candidates_k / --candidates_among / --candidates_diversity / --candidates_pool, checked before the first
    training step -> the ids of --candidates_among (int64 CPU, sorted, distinct), or None."""
    among_path = getattr(args, "candidates_among", None)
    lam, pool = getattr(args, "candidates_diversity", None), getattr(args, "candidates_pool", None)
    if among_path and not args.candidates_out:
        raise ValueError("--candidates_among restricts the --candidates_out file: give --candidates_out too")
    for flag, v in (("--candidates_diversity", lam), ("--candidates_pool", pool)):
        if v is not None and not args.candidates_out:
            raise ValueError(f"{flag} diversifies the --candidates_out file: give --candidates_out too")
    if pool is not None and lam is None:
        raise ValueError("--candidates_pool is the pool of a diversified --candidates_out file: give --candidates_diversity too")
    if not args.candidates_out:
        return None
    among = None if not among_path else recommend.read_among(among_path, n_items)
    rankable = n_items if among is None else among.numel()
    K = recommend.check_k(args.candidates_k, n_items) if among is None else \
        recommend.check_k(args.candidates_k, rankable, "|--candidates_among|")
    if recommend.check_diversity(lam) is not None and pool is not None:
        recommend.check_pool(pool, K, min(recommend.MAX_K, rankable), f"--candidates_pool: at most {recommend.MAX_K} and at most the "
                                                                      f"{rankable} rankable ids")
    return among


def check_rerank_flags(args, trainer):
    """--rerank_in / --rerank_out / --rerank_k, checked before the first training step -> (the candidate array, K), or (None, None)."""
    if not args.rerank_in and not args.rerank_out:
        return None, None
    if not (args.rerank_in and args.rerank_out):
        raise ValueError("--rerank_in and --rerank_out go together: the candidate file to re-rank and the file to write")
    if trainer.masked_mode:
        raise ValueError("--rerank_in needs a fixed model: not with --mask / --mask_rate > 0 / --drop_rate > 0")
    recommend.check_engine(trainer.hot)
    cand = recommend.read_candidates(args.rerank_in, trainer.n_users, trainer.n_items)
    K = int(cand.shape[1]) if args.rerank_k is None else args.rerank_k
    recommend.check_rerank_k(K)
    return cand, K


def check_groups_flags(args, trainer):
    """--groups_in / --groups_out / --groups_k / --groups_agg, checked before the first training step -> the groups ((rowptr, col) of
    recommend.groups_csr), or None."""
    g_in, g_out = getattr(args, "groups_in", None), getattr(args, "groups_out", None)
    if not g_in and not g_out:
        return None
    if not (g_in and g_out):
        raise ValueError("--groups_in and --groups_out go together: the file of groups and the file to write")
    if trainer.masked_mode:
        raise ValueError("--groups_in needs a fixed model: not with --mask / --mask_rate > 0 / --drop_rate > 0")
    recommend.check_engine(trainer.hot)
    recommend.check_k(getattr(args, "groups_k", 10), trainer.n_items)
    recommend.check_agg(getattr(args, "groups_agg", "mean"))
    return recommend.read_groups(g_in, trainer.n_users)


if __name__ == "__main__":
    main()
