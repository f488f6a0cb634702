"""Host mirror of Stract's recall ranking stage (RankingPipeline::recall_stage, core/src/ranking/pipeline/stages/recall.rs:303-333,
pipeline/mod.rs:136-162) over the recall webpages of MultiFieldSignalComputer.ranking_webpages.

A page is (signals, score, boost): `signals` maps a SignalEnum name to (value, score); the page starts with the initial total
as its score and SignalComputer::boosts as its boost (recall.rs:198-217).  Each stage computes, then `update_scores` re-sums
sum(score * coefficient) over the present signals in SignalEnum order (scorers/mod.rs:50-56), then `rank` sorts the pages
stably by boost * score, descending.  The InboundSimilarity modifier multiplies the boost by value + 8 and re-ranks without
re-summing.  With a model (stract_b200.lambdamart.LambdaMART, the reference's `lambda_model_path`) the LambdaMART stage follows:
the top 20 pages are predicted on the device, re-summed and ranked, unless the query's offset is above 20.  The embeddings
themselves and the precision stage need models the reference does not ship and are not mirrored."""
import numpy as np

from .bm25 import CORE_SIGNALS, NUMERIC_SIGNALS

# SignalEnum in declaration order (core/src/ranking/signals/mod.rs:108-155): the iteration order of EnumMap<SignalEnum, _>
SIGNAL_ENUM = ["Bm25F", "Bm25Title", "TitleCoverage", "Bm25TitleBigrams", "Bm25TitleTrigrams", "Bm25CleanBody", "CleanBodyCoverage",
               "Bm25CleanBodyBigrams", "Bm25CleanBodyTrigrams", "Bm25StemmedTitle", "Bm25StemmedCleanBody", "Bm25AllBody", "Bm25Keywords",
               "Bm25BacklinkText", "IdfSumUrl", "IdfSumSite", "IdfSumDomain", "IdfSumSiteNoTokenizer", "IdfSumDomainNoTokenizer",
               "IdfSumDomainNameNoTokenizer", "IdfSumDomainIfHomepage", "IdfSumDomainNameIfHomepageNoTokenizer",
               "IdfSumDomainIfHomepageNoTokenizer", "IdfSumTitleIfHomepage", "CrossEncoderSnippet", "CrossEncoderTitle", "HostCentrality",
               "HostCentralityRank", "PageCentrality", "PageCentralityRank", "IsHomepage", "FetchTimeMs", "UpdateTimestamp",
               "TrackerScore", "Region", "QueryCentrality", "InboundSimilarity", "LambdaMart", "UrlDigits", "UrlSlashes", "LinkDensity",
               "TitleEmbeddingSimilarity", "KeywordEmbeddingSimilarity", "HasAds", "MinTitleSlop", "MinCleanBodySlop"]

# default coefficients of the signals outside CoreSignalEnum (core/src/ranking/signals/non_core/*.rs)
NON_CORE_COEFFICIENTS = {"QueryCentrality": 0.0, "InboundSimilarity": 0.25, "LambdaMart": 10.0, "MinTitleSlop": 0.1, "MinCleanBodySlop": 0.1,
                         "CrossEncoderSnippet": 0.17, "CrossEncoderTitle": 0.17, "TitleEmbeddingSimilarity": 0.01,
                         "KeywordEmbeddingSimilarity": 0.01}

U32_MAX = 0xFFFFFFFF
INBOUND_SIMILARITY_SMOOTHING = 8.0   # modifiers/inbound_similarity.rs


def default_coefficients():
    """SignalCoefficients::default(): every SignalEnum's default coefficient."""
    c = {name: coef for name, _k, _f, _s, coef in CORE_SIGNALS}
    c.update({name: coef for name, _k, _d, coef in NUMERIC_SIGNALS})
    c.update(NON_CORE_COEFFICIENTS)
    return c


def min_slop_two_positions(pos_a, pos_b):
    """term_distance.rs:23-46, the two-cursor walk"""
    cur_min, ca, cb = U32_MAX, 0, 0
    while ca < len(pos_a) and cb < len(pos_b):
        a, b = pos_a[ca], pos_b[cb]
        if b > a:
            cur_min = min(b - a, cur_min)
            ca += 1
        else:
            cb += 1
    return cur_min


def min_slop(positions):
    """term_distance.rs:48-54: the max over consecutive lists (tuple_windows), u32::MAX with fewer than 2"""
    pairs = [min_slop_two_positions(a, b) for a, b in zip(positions, positions[1:])]
    return max(pairs) if pairs else U32_MAX


def score_slop(slop):
    return 1.0 / (float(slop) + 1.0)


class Page:
    """One ranking webpage: `signals` {SignalEnum name: (value, score)}, `score` (unboosted), `boost`, `key` the caller's id."""

    def __init__(self, key, signals, score, boost):
        self.key, self.signals, self.score, self.boost = key, dict(signals), float(score), float(boost)

    def total(self):
        return self.boost * self.score


def pages_from_webpages(wp, q, docs, n, initial_totals):
    """The pages of query q from ranking_webpages' result `wp` (its op names are the signals), the initial totals
    (the top-k entry point's f64 totals, WebpagePointer.score.total) and the documents as keys.  MinTitleSlop / MinCleanBodySlop
    are not signals yet: recall_stage computes them from min_slop."""
    out = []
    for i in range(n):
        sig = {name: (float(wp.values[q, i, o]), float(wp.scores[q, i, o])) for o, name in enumerate(wp.names)}
        p = Page(int(docs[i]), sig, initial_totals[i], wp.boosts[q, i])
        p.min_slop = (int(wp.min_slop[q, i, 0]), int(wp.min_slop[q, i, 1]))
        out.append(p)
    return out


def update_scores(pages, coefficients):
    """FullRankingStage::update_scores: per page, fold from 0.0 over its present signals in SignalEnum order of
    acc + score * coefficient -- sequential over the signals, vectorised over the pages, two roundings per step (no FMA)."""
    if not pages:
        return
    acc = np.zeros(len(pages))
    for name in SIGNAL_ENUM:
        have = np.array([name in p.signals for p in pages])
        if not have.any():
            continue
        sc = np.array([p.signals[name][1] if name in p.signals else 0.0 for p in pages])
        prod = sc * np.float64(coefficients.get(name, 0.0))
        acc = np.where(have, acc + prod, acc)
    for p, a in zip(pages, acc):
        p.score = float(a)


def rank(pages):
    """sort_by(b.score().partial_cmp(&a.score())): stable, descending boost * score"""
    pages.sort(key=lambda p: -p.total())


def _stage(pages, coefficients, compute):
    compute(pages)
    update_scores(pages, coefficients)
    rank(pages)


LAMBDAMART_TOP = 20   # Top::Limit(20), pipeline/scorers/lambdamart.rs:38-40


def recall_stage(pages, coefficients, inbound, lambdamart=None, offset=0):
    """RankingPipeline::recall_stage for one query: recall_stage_batch with one query."""
    return recall_stage_batch([pages], coefficients, inbound, lambdamart, offset)[0]


def recall_stage_batch(pages_per_query, coefficients, inbound, lambdamart=None, offset=0):
    """RankingPipeline::recall_stage per query: TitleDistanceScorer, BodyDistanceScorer, the two embedding stages (no dual
    encoder: they insert nothing, embedding.rs:122-125, but still re-sum and rank), InboundScorer with `inbound` {page key: score}
    (e.g. Webgraph.inbound_similarity), the InboundSimilarity modifier, then with a `lambdamart` model the LambdaMART stage over
    each query's top 20 (pipeline/mod.rs:136-162: skipped when `offset`, page * num_results, is above 20), predicted for every
    query in one device call.  Pages carry `min_slop` (Title, CleanBody).  Returns each query's pages in their final order."""
    coefficients = dict(coefficients)
    out = [_recall_host_stages(list(pages), coefficients, inbound) for pages in pages_per_query]
    if lambdamart is None or offset > LAMBDAMART_TOP:
        return out
    tops = [pages[:LAMBDAMART_TOP] for pages in out]
    flat = [p for top in tops for p in top]
    scores = lambdamart.predict(lambdamart.feature_rows(flat)) if flat else []
    for p, s in zip(flat, scores):
        p.signals["LambdaMart"] = (float(s), float(s))   # SignalCalculation::new_symmetrical
    for pages, top in zip(out, tops):
        update_scores(top, coefficients)
        rank(top)
        pages[:len(top)] = top
    return out


def _recall_host_stages(pages, coefficients, inbound):
    """the stages before LambdaMART, in place on `pages`"""
    def distance(field, name):
        def compute(ps):
            for p in ps:
                v = float(p.min_slop[field])
                p.signals[name] = (v, score_slop(v))
        return compute

    _stage(pages, coefficients, distance(0, "MinTitleSlop"))
    _stage(pages, coefficients, distance(1, "MinCleanBodySlop"))
    _stage(pages, coefficients, lambda ps: None)   # TitleEmbeddings
    _stage(pages, coefficients, lambda ps: None)   # KeywordEmbeddings

    def inbound_scorer(ps):
        for p in ps:
            s = float(inbound[p.key])
            p.signals["InboundSimilarity"] = (s, s)
    _stage(pages, coefficients, inbound_scorer)
    for p in pages:   # modifiers::InboundSimilarity: boost *= value + 8; no re-sum
        v = p.signals["InboundSimilarity"][0] if "InboundSimilarity" in p.signals else 0.0
        p.boost = p.boost * (v + INBOUND_SIMILARITY_SMOOTHING)
    rank(pages)
    return pages
