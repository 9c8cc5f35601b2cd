"""Golden data of the training negatives: a small seeded raw MIND behaviours file and what the reference's own
preprocessing makes of it.

    python oracle/make_golden_negsample.py /path/to/news-recommendation/src

writes tests/golden/negsample/{behaviors.tsv, news_parsed.tsv}, then runs the reference's parse_behaviors (src/
data_preprocess.py) on behaviors.tsv with `random` seeded, which writes user2int.tsv and behaviors_parsed.tsv next to it.
negative_sampling_ratio is the reference NRMS config's (K = 2).  The impressions cover: no positive, fewer negatives than
K, more positives than N // K, many positives and negatives, labels in shuffled order; the histories: empty, exactly 50,
longer than 50 (num_clicked_news_a_user); several impressions of one user.  The reference imports swifter and
nltk.tokenize at module level for its news parser; the balancing step uses neither, so both are stubbed.  Only this
script needs the reference.  Under pandas 3 the reference's chained fillna(' ', inplace=True) no longer reaches the
frame, so an empty history stays an empty field in behaviors_parsed.tsv (read it with keep_default_na=False).
"""
import os
import random
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "negsample")
N_NEWS, T, TA = 40, 20, 50


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
    # (positives, negatives, history length); 0 history -> an empty field, as MIND writes it
    shapes = [(1, 4, 12), (0, 6, 3), (2, 1, 50), (1, 0, 60), (3, 4, 0), (1, 1, 7), (2, 9, 51), (5, 3, 20), (1, 2, 1),
              (4, 30, 33), (0, 1, 5), (2, 2, 0), (1, 25, 44), (6, 13, 2), (1, 3, 9), (3, 7, 70), (2, 5, 16), (1, 12, 50)]
    users = ["U7", "U3", "U7", "U19", "U42", "U5", "U7", "U26", "U8", "U31", "U42", "U11", "U2", "U3", "U60", "U9", "U7", "U13"]
    with open(os.path.join(out, "behaviors.tsv"), "w") as f:
        for n, ((P, N, h), u) in enumerate(zip(shapes, users)):
            items = [f"{rng.choice(news)}-1" for _ in range(P)] + [f"{rng.choice(news)}-0" for _ in range(N)]
            rng.shuffle(items)
            f.write(f"{n + 1}\t{u}\t11/{n % 28 + 1}/2019 9:{n:02d}:00 AM\t{hist(h)}\t{' '.join(items)}\n")


def main(reference_src):
    write_fixture(OUT)
    for name in ("swifter", "nltk", "nltk.tokenize"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["nltk.tokenize"].word_tokenize = lambda s: s.split()
    sys.path.insert(0, os.path.abspath(reference_src))
    os.environ.setdefault("MODEL_NAME", "NRMS")
    import pandas as pd
    pd.options.future.infer_string = False  # the reference stores ints into its user column
    import data_preprocess
    assert data_preprocess.config.negative_sampling_ratio == 2
    random.seed(20261018)
    data_preprocess.parse_behaviors(os.path.join(OUT, "behaviors.tsv"), os.path.join(OUT, "behaviors_parsed.tsv"),
                                    os.path.join(OUT, "user2int.tsv"))
    print("wrote", OUT)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ["NEWSREC_REFERENCE_SRC"])
