"""Command-line flags of the reference (utility/parser.py:4-56), same names, types and defaults.

Table-driven restatement: typed tables of (default, meaning) instead of one add_argument call per flag.
`--mask` keeps the reference's `type=bool` quirk (any non-empty string is True, parser.py:39).
`--dataset netflix|movielens` are accepted as aliases of the on-disk directory names
(README.md:80-82 documents the short names; main.py:69-72 only handles the long ones).
"""
import argparse

# name -> (default, what it controls).  Grouped by how argparse converts the value; defaults are the reference's.
_INT = {
    "seed": (2022, "seed of random / numpy / torch"),
    "verbose": (5, "evaluate every this many epochs"),
    "epoch": (1000, "maximum number of epochs"),
    "embed_size": (64, "width d of the id embeddings and of every projected feature"),
    "early_stopping_patience": (7, "evaluations without a better recall@20 before stopping"),
    "sparse": (1, "unused by LLMRec (kept for CLI compatibility)"),
    "gpu_id": (0, "CUDA device"),
    "batch_size": (1024, "sampled interactions per step (augmented edges come on top)"),
    "layers": (1, "unused by LLMRec: the layer count is len(weight_size)"),
}
_FLOAT = {
    "sc": (1.0, "unused by LLMRec"),
    "feat_reg_decay": (1e-5, "weight of the squared-norm regulariser on the propagated image/text features"),
    "lr": (0.0001, "AdamW learning rate"),
    "de_lr": (0.0002, "learning rate of the (unused) decoder optimiser"),
    "weight_decay": (1e-4, "unused: AdamW runs with torch's default 0.01"),
    "drop_rate": (0.0, "dropout on the projected side features (> 0 runs the eager mask / dropout branch, Trainer._train_batch_masked)"),
    "mask_rate": (0.0, "share of nodes whose features are overwritten with the column mean (> 0 runs the eager mask / dropout branch)"),
    "user_cat_rate": (2.8, "fusion weight of the normalised user-profile term"),
    "item_cat_rate": (0.005, "fusion weight of each normalised item-attribute term"),
    "model_cat_rate": (0.02, "fusion weight of the normalised image and text terms"),
    "de_drop1": (0.31, "unused"),
    "de_drop2": (0.5, "unused"),
    "aug_mf_rate": (0.012, "weight of the attribute BPR heads"),
    "prune_loss_drop_rate": (0.71, "share of the batch dropped by prune_loss (the least negative log-sigmoids)"),
    "mm_mf_rate": (0.0001, "weight of the image and text BPR heads"),
    "att_re_rate": (0.00000, "weight of the attribute-restoration loss (mask branch)"),
    "alpha_l": (2, "exponent of the sce restoration loss (mask branch)"),
    "aug_sample_rate": (0.1, "share of the batch's users that contribute an LLM-augmented edge"),
    "mf_emb_rate": (0.0, "unused"),
}
_OPTIONAL_TEXT = {                     # nargs="?": python-literal strings are eval()ed by the trainer, like upstream
    "data_path": ("./data/", "directory that holds the dataset directories"),
    "dataset": ("netflix", "netflix | movielens, or the on-disk directory name"),
    "regs": ("[1e-5,1e-5,1e-2]", "regs[0] scales the reciprocal-norm embedding term"),
    "weight_size": ("[64, 64]", "one entry per propagation layer"),
    "mess_dropout": ("[0.1, 0.1]", "unused by LLMRec"),
    "norm_type": ("sym", "unused by LLMRec"),
    "Ks": ("[10, 20, 50]", "cut-offs of recall / precision / hit / ndcg"),
    "test_flag": ("part", "part = top-K metrics; full = the same plus the per-user ROC-AUC over every candidate"),
    "cf_model": ("lightgcn", "name used in the log file name"),
}
_TEXT = {
    "title": ("try_to_draw_line", "free text"),
    "point": ("", "free text"),
    "feat_loss_type": ("sce", "mse | sce (mask branch)"),
}


def _reference_flags():
    rows = [(k, dict(type=int, default=v, help=h)) for k, (v, h) in _INT.items()]
    rows += [(k, dict(type=float, default=v, help=h)) for k, (v, h) in _FLOAT.items()]
    rows += [(k, dict(nargs="?", default=v, help=h)) for k, (v, h) in _OPTIONAL_TEXT.items()]
    rows += [(k, dict(type=str, default=v, help=h)) for k, (v, h) in _TEXT.items()]
    rows.append(("debug", dict(action="store_true", help="do not write ./logs/")))
    rows.append(("mask", dict(type=bool, default=False, help="bool('...'): ANY non-empty value switches the mask branch on (upstream quirk)")))
    return rows


_FLAGS = _reference_flags()

# GPU-side extras (not in the reference; all optional)
_EXTRA = [
    ("proj_mode", dict(default="3xtf32", choices=["3xtf32", "tf32", "fp32"], help="tensor-core mode of the projection / scoring GEMMs")),
    ("cuda_graph", dict(type=int, default=1, help="replay the training step from a CUDA graph (1) or launch eagerly (0)")),
    ("host_sampler", dict(default="native", choices=["native", "python"], help="bit-identical C sampler or the reference's Python loops")),
    ("hoist_side", dict(type=int, default=0, help="1: precompute the propagation of the constant side features once (ui.X, iu.ui.X) and project only the "
                                                   "batch's rows per step (SURVEY.md 8f-3); same results within the golden tolerances; off automatically "
                                                   "when drop_rate > 0 or the mask branch is on")),
    ("device_sampler", dict(type=int, default=0, choices=[0, 1, 2], help="0: the reference's batches, drawn on the host (default); 1: batches drawn on the GPU from their own RNG stream (same distributions, other batches, SURVEY.md 8f-1); 2: the reference's exact batches, drawn on the GPU from device copies of `random` / `np.random`")),
    ("feat_dtype", dict(default="fp32", choices=["fp32", "bf16", "int8"], help="element type the side-feature tables (image, text, user profile, "
                                                                      "attributes) are kept in: bf16 rounds them once (round-to-nearest-even) "
                                                                      "when the model is built and halves their memory and projection reads; "
                                                                      "int8 quantizes each row once to int8 values and a power-of-two scale "
                                                                      "(every stored value an exact bf16), a quarter of the fp32 bytes; "
                                                                      "the projections are then exact on the rounded tables. Not with the mask branch")),
    ("deterministic", dict(type=int, default=0, help="1: bit-reproducible training steps -- the loss heads accumulate their row gradients in a fixed "
                                                     "order (heads, then batch positions, pos before neg) instead of with float atomics, so one "
                                                     "--seed gives one model. Not with --proj_mode fp32, the mask / dropout branch or the sharded engines")),
    ("save_dir", dict(default=None, help="directory for checkpoints: last.pt after every --save_every epochs (after the evaluation), best.pt whenever "
                                         "recall@Ks[1] improves. Nothing is written without it. Not with the mask / dropout branch")),
    ("save_every", dict(type=int, default=1, help="epochs between two writes of last.pt (with --save_dir)")),
    ("resume", dict(default=None, help="checkpoint to continue from: parameters, AdamW state, RNG streams and the position in the training loop are "
                                       "put back before the first step, so training goes on as if it had never stopped")),
    ("eval_only", dict(type=int, default=0, help="1: run no training step, evaluate the model of --resume once on the test users")),
    ("candidates_out", dict(default=None, help="when the run ends (after training, or after --eval_only 1), write every user's top --candidates_k "
                                               "items over the whole catalog, nothing excluded, as the pickled CPU int64 tensor [n_users x K] "
                                               "the augmentation stage reads (data/<dataset>/candidate_indices). Not with the mask / dropout branch")),
    ("candidates_k", dict(type=int, default=10, help="list length of --candidates_out (1..64, at most n_items)")),
    ("candidates_among", dict(default=None, help="restrict --candidates_out to these items: a pickled 1-D integer tensor, ndarray or list "
                                                 "of item ids (order and repeats do not matter); each user's list is then the top "
                                                 "--candidates_k of these ids (at most their number). Needs --candidates_out")),
    ("candidates_diversity", dict(type=float, default=None, help="diversify --candidates_out: lambda in [0, 1]; each user's list is picked "
                                                                 "greedily from the user's top --candidates_pool items, each time the item "
                                                                 "with the largest lambda * score - (1 - lambda) * (its largest cosine to an "
                                                                 "item already picked); 1 = the plain top list. Needs --candidates_out")),
    ("candidates_pool", dict(type=int, default=None, help="pool size of --candidates_diversity (--candidates_k..64, at most the number of "
                                                          "rankable items; default the smaller of 64 and that number)")),
    ("rerank_in", dict(default=None, help="when the run ends, re-rank a candidate file with this model: a pickled 2-D integer tensor or "
                                          "ndarray [n_users x C], row u = user u's candidates, -1 = padding (the --candidates_out / "
                                          "candidate_indices format, so a file made by another model can be reordered by this one). "
                                          "Needs --rerank_out. Not with the mask / dropout branch")),
    ("rerank_out", dict(default=None, help="where --rerank_in's rows go, re-ranked by (score desc, id asc), nothing excluded, repeats kept "
                                           "once: the pickled CPU int64 tensor [n_users x --rerank_k], padded with -1, written atomically")),
    ("rerank_k", dict(type=int, default=None, help="list length of --rerank_out (1..1024; default: the width C of --rerank_in)")),
    ("groups_in", dict(default=None, help="when the run ends, recommend for groups of users who choose together: a pickled list of "
                                          "trained-user-id lists, one per group (1..64 distinct members each; repeats and order do not "
                                          "matter). Needs --groups_out. Not with the mask / dropout branch")),
    ("groups_out", dict(default=None, help="where --groups_in's lists go: each group's top --groups_k items under --groups_agg, every "
                                           "member's training items excluded, as the pickled CPU int64 tensor [n_groups x K], padded "
                                           "with -1, written atomically")),
    ("groups_k", dict(type=int, default=10, help="list length of --groups_out (1..64, at most n_items)")),
    ("groups_agg", dict(default="mean", choices=["mean", "min", "max"], help="group score of --groups_out: the mean of the members' "
                                                                             "scores, the least misery (min) or the most pleasure (max)")),
]

DATASET_ALIASES = {"netflix": "netflix_valid_item", "movielens": "preprocessed_raw_MovieLens", "movieLens": "preprocessed_raw_MovieLens"}


def build_parser():
    ap = argparse.ArgumentParser(description="")
    for name, kw in _FLAGS + _EXTRA:
        ap.add_argument("--" + name, **kw)
    return ap


def parse_args(argv=None):
    """parse_args() -> Namespace (reference: utility/parser.py:4).  Unknown flags are an error."""
    return build_parser().parse_args(argv)


def resolve_dataset_dir(data_path, dataset):
    """Directory that holds the dataset: the literal name if it exists, else its alias."""
    import os
    first = os.path.join(data_path, dataset)
    if os.path.isdir(first):
        return first
    alias = DATASET_ALIASES.get(dataset)
    if alias and os.path.isdir(os.path.join(data_path, alias)):
        return os.path.join(data_path, alias)
    return first
