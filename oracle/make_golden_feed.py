"""Golden data of the training feed: a small seeded parsed-MIND fixture and the batches the reference's own BaseDataset +
default_collate make of it.

    python oracle/make_golden_feed.py /path/to/news-recommendation/src

writes tests/golden/feed/news_parsed.tsv, tests/golden/feed/behaviors_parsed.tsv and tests/golden/feed.npz.  The fixture
has nonzero entity ids, an empty history, histories of exactly 50 and of 60 news, a news id repeated within a history and
several rows of one user.  For every family the reference's dataset is built with that family's config class (its news
attributes and records, num_clicked_news_a_user = 50) and ONE batch of all rows in a fixed order is collated.  Keys of
feed.npz, per family F: F.order (B,), F.clicked_news.<attr> (H, B[, L]), F.candidate_news.<attr> (C, B[, L]),
F.clicked (C, B), F.user / F.clicked_news_length (B,) when the family records them.  Only this script needs the reference.
"""
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")
FAMILIES = ("NRMS", "NAML", "LSTUR", "TANR", "Exp1", "HiFiArk", "DKN")
N_NEWS, T, TA, C, H = 30, 20, 50, 5, 50


def write_fixture(out):
    rng = random.Random(20261018)
    os.makedirs(out, exist_ok=True)

    def ids(n, length, hi):
        k = rng.randint(1, n)
        return [rng.randint(1, hi) for _ in range(k)] + [0] * (length - k)

    with open(os.path.join(out, "news_parsed.tsv"), "w") as f:
        f.write("id\tcategory\tsubcategory\ttitle\tabstract\ttitle_entities\tabstract_entities\n")
        for i in range(N_NEWS):
            f.write(f"N{100 + i}\t{rng.randint(1, 17)}\t{rng.randint(1, 60)}\t{ids(T, T, 999)}\t{ids(TA, TA, 999)}\t"
                    f"{ids(T, T, 400)}\t{ids(TA, TA, 400)}\n")
    news = [f"N{100 + i}" for i in range(N_NEWS)]
    hist = lambda n: " ".join(rng.choice(news) for _ in range(n))
    histories = [
        " ",                                       # no history: 50 padding news, clicked_news_length 0
        hist(50),                                  # exactly num_clicked_news_a_user
        hist(60),                                  # truncated to its first 50
        " ".join(["N105", "N117", "N105", "N120", "N105"]),  # a news id repeated within a history
        hist(1), hist(49), hist(51), hist(7), hist(23), hist(60), hist(2), hist(34),
    ]
    users = [11, 7, 42, 7, 3, 7, 19, 42, 5, 26, 8, 31]  # user 7 and user 42 own several rows
    with open(os.path.join(out, "behaviors_parsed.tsv"), "w") as f:
        f.write("user\tclicked_news\tcandidate_news\tclicked\n")
        for u, h in zip(users, histories):
            cand = " ".join(rng.choice(news) for _ in range(C))
            f.write(f"{u}\t{h}\t{cand}\t{' '.join(['1'] + ['0'] * (C - 1))}\n")
    return len(histories)


def main(reference_src):
    out = os.path.join(GOLDEN, "feed")
    R = write_fixture(out)
    sys.path.insert(0, os.path.abspath(reference_src))
    import pandas as pd
    pd.options.future.infer_string = False
    import torch
    from torch.utils.data import default_collate
    import config as refconfig
    import dataset as refdataset
    order = np.random.default_rng(7).permutation(R)
    arrays = {}
    for fam in FAMILIES:
        cfg = getattr(refconfig, f"{fam}Config")
        assert cfg.num_clicked_news_a_user == H and cfg.num_words_title == T and cfg.num_words_abstract == TA
        refdataset.config = cfg  # the module-level config the reference dataset reads
        ds = refdataset.BaseDataset(os.path.join(out, "behaviors_parsed.tsv"), os.path.join(out, "news_parsed.tsv"))
        batch = default_collate([ds[int(i)] for i in order])
        arrays[f"{fam}.order"] = order.astype(np.int64)
        for key in ("clicked_news", "candidate_news"):
            for attr in cfg.dataset_attributes["news"]:
                arrays[f"{fam}.{key}.{attr}"] = torch.stack([slot[attr] for slot in batch[key]]).numpy()
        arrays[f"{fam}.clicked"] = torch.stack(batch["clicked"]).numpy()
        for rec in cfg.dataset_attributes["record"]:
            arrays[f"{fam}.{rec}"] = batch[rec].numpy()
    np.savez_compressed(os.path.join(GOLDEN, "feed.npz"), **arrays)
    print("wrote", out, "and feed.npz with", len(arrays), "arrays")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ["NEWSREC_REFERENCE_SRC"])
