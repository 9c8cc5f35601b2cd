"""Knob surface of the drop-in: the attribute names, defaults and `MODEL_NAME` selection that the
reference's callers read (reference src/config.py:3-106; train.py:9,19; dataset.py:6,11).

The values are the reference defaults; the classes are generated from one table so that the file is a
restatement of the knob surface, not a copy of the reference source.
"""
import os

model_name = os.environ.get("MODEL_NAME", "NRMS")
SUPPORTED_MODELS = ("NRMS", "NAML", "LSTUR", "TANR", "Exp1", "HiFiArk", "DKN")  # the hot-path scope of this build (SURVEY.md section 8)
if model_name not in SUPPORTED_MODELS:
    raise AssertionError(f"MODEL_NAME={model_name!r}: this build accelerates {SUPPORTED_MODELS} only")

_COMMON = {
    # training loop (read by the reference's train.py / evaluate.py, not by the kernels)
    "num_epochs": 2, "num_batches_show_loss": 100, "num_batches_validate": 1000, "batch_size": 128,
    "learning_rate": 0.0001, "num_workers": 4,
    # data shapes
    "num_clicked_news_a_user": 50, "num_words_title": 20, "num_words_abstract": 50,
    "word_freq_threshold": 1, "entity_freq_threshold": 2, "entity_confidence_threshold": 0.5,
    "negative_sampling_ratio": 2,
    # regularisation
    "dropout_probability": 0.2,
    # vocabulary sizes (MIND-small; edit after preprocessing exactly as with the reference)
    "num_words": 1 + 70975, "num_categories": 1 + 274, "num_entities": 1 + 12957, "num_users": 1 + 50000,
    # widths
    "word_embedding_dim": 300, "category_embedding_dim": 100, "entity_embedding_dim": 100,
    "query_vector_dim": 200,
}
BaseConfig = type("BaseConfig", (), dict(_COMMON, __doc__="General configuration shared by all models"))

# window_size: 1 to 4 (the conv GEMMs take at most 4 taps); building a CNN model with any other window raises NewsrecError.
# The reference asserts an odd window in LSTUR, TANR and Hi-Fi Ark; this build runs 2 and 4 there as NAML's conv does
_CNN = {"num_filters": 300, "window_size": 3}
_PER_MODEL = {
    # precision is an extension knob of this build (not in the reference; DESIGN.md section 4):
    #   precision "accurate" (default): V / attention probabilities / context as hi/lo bf16 pairs and an fp32-accurate user
    #   encoder -- logits within 1e-3 of the fp32 oracle on bf16-rounded weights (the blueprint's tolerance); "fast": every
    #   activation stored bf16 (~6e-3).  Shapes the title-level attention kernel does not cover fall back to "fast".
    "NRMS": dict(dataset_attributes={"news": ["title"], "record": []}, num_attention_heads=15,
                 precision=os.environ.get("NEWSREC_PRECISION", "accurate")),
    "NAML": dict(dataset_attributes={"news": ["category", "subcategory", "title", "abstract"], "record": []}, **_CNN),
    "LSTUR": dict(dataset_attributes={"news": ["category", "subcategory", "title"],
                                      "record": ["user", "clicked_news_length"]},
                  long_short_term_method="ini", masking_probability=0.5,
                  # extension knob (see NRMS): "accurate" = conv output and GRU input as hi/lo bf16 pairs (1e-3 tolerance of the
                  # blueprint for both long/short-term methods), "fast" = plain bf16 storage (ini: 1.8e-3)
                  precision=os.environ.get("NEWSREC_PRECISION", "accurate"), **_CNN),
    "TANR": dict(dataset_attributes={"news": ["category", "title"], "record": []},
                 topic_classification_loss_weight=0.1, **_CNN),
    # the reference leaves "abstract" as a TODO for Exp1; this build raises if it is configured (DESIGN.md section 6).
    # precision as NRMS: "accurate" also keeps the stacked views in front of final_attention as hi/lo bf16 pairs
    "Exp1": dict(dataset_attributes={"news": ["category", "subcategory", "title"], "record": []}, num_attention_heads=15,
                 ensemble_factor=1, precision=os.environ.get("NEWSREC_PRECISION", "accurate")),
    # plain bf16 storage in the news encoder meets the 1e-3 contract (DESIGN.md section 4): no precision knob
    "HiFiArk": dict(dataset_attributes={"news": ["title"], "record": []}, num_pooling_heads=5, regularizer_loss_weight=0.1, **_CNN),
    # plain bf16 storage meets the 1e-3 contract (DESIGN.md section 4); use_context=True raises (context embeddings unavailable)
    "DKN": dict(dataset_attributes={"news": ["title", "title_entities"], "record": []}, num_filters=50, window_sizes=[2, 3, 4],
                use_context=False),
}
for _name, _knobs in _PER_MODEL.items():
    globals()[f"{_name}Config"] = type(f"{_name}Config", (BaseConfig,), dict(_knobs))
assert LSTURConfig.long_short_term_method in ("ini", "con")  # noqa: F821
del _name, _knobs
