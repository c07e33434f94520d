"""Generation and criterion metrics of the validators, written for this package (sacremoses and sacrebleu are not
dependencies of it), with the behaviour of the reference's metrics:

  Wer / CER                  neurst/metrics/wer.py: edit operations with its tie order, percent keys; its text
                             normalisation (lowercase, contractions, punctuation) with the Moses normaliser as the identity
  BLEU: tok_bleu             neurst/metrics/bleu.py's corpus BLEU (no smoothing) over XML-unescaped text
        sacre_bleu / detok   sacrebleu.corpus_bleu(tokenize="13a") with its default `exp` smoothing
  CriterionMetric            LabelSmoothedCrossEntropy.reduce_metrics / as_metric (lower is better)

Hypotheses and references reach the metrics as `ids_to_text` of token ids, i.e. text that the recipe's transcript pipeline
already Moses-tokenised; the Moses tokenizer is therefore taken as the identity (DESIGN.md, "Validation").  `chrf`, several
references per sentence and the languages whose BLEU needs a character, Thai or MeCab tokenizer are refused.
"""
import math
import re
from collections import Counter

import numpy as np

# ------------------------------------------------------------------------------------------------ text normalisation
CHARACTER_LANGUAGES = ("zh", "ja")               # WER counts characters (CER) for these
# the characters the WER normalisation turns into spaces (the reference's punctuation set, ASCII and CJK)
WER_PUNCTUATION = re.compile("[%s]" % re.escape(",.!();:、?-+=\"/><《》[]，。：；「」【】{}`@#$%^&*"))


def normalize_for_wer(language, text):
    """Lowercase; outside zh / ja rejoin the contractions the Moses tokenizer splits ("it' s " -> "it's "); punctuation
    to spaces; single spaces, none at the ends."""
    text = text.lower()
    if language not in CHARACTER_LANGUAGES:
        for suffix in ("s", "ve", "m", "t", "re"):
            text = text.replace("' %s " % suffix, "'%s " % suffix)
    return " ".join(WER_PUNCTUATION.sub(" ", text).split())


# ------------------------------------------------------------------------------------------------ metric base
class Metric:
    """neurst/metrics/metric.py: `flag` names the value that ranks results; greater_or_eq(a, b) is True when a is at
    least as good as b."""

    def __init__(self):
        self.flag = self.__class__.__name__

    def greater_or_eq(self, result1, result2):
        return self.get_value(result1) >= self.get_value(result2)

    def get_value(self, result):
        if isinstance(result, dict) and self.flag in result:
            return result[self.flag]
        return result

    def __call__(self, hypothesis, groundtruth):
        res = self.call(hypothesis, groundtruth)
        return res if isinstance(res, dict) else {self.flag: res}


class CriterionMetric(Metric):
    """LabelSmoothedCrossEntropy.as_metric(): MetricWrapper(flag="NLL", greater_is_better=False), with reduce_metrics
    over the summed criterion outputs."""

    def __init__(self):
        super().__init__()
        self.flag = "NLL"

    def greater_or_eq(self, result1, result2):
        return not super().greater_or_eq(result1, result2)

    @staticmethod
    def reduce(nll_sum, n_samples, n_tokens):
        """NLL per sentence, PPL = 2 ** (NLL per token): the base-2 exponent is the reference's."""
        return {"NLL": nll_sum / n_samples, "PPL": 2. ** (nll_sum / n_tokens)}

    def call(self, hypothesis, groundtruth):
        raise NotImplementedError("the criterion metric is reduced from loss sums (CriterionMetric.reduce)")


# ------------------------------------------------------------------------------------------------ WER / CER
def _wer(ref, hypo):
    """wer.py:21-34: (substitutions, insertions, deletions) of the first minimum in the order substitution, insertion,
    deletion (`min(..., key=np.sum)` keeps the first of equal sums).  The same recurrence on integer tuples, one row at a
    time: the reference's per-cell NumPy operations take seconds on a dev set."""
    prev = [(0, j, 0) for j in range(len(hypo) + 1)]
    for r, rw in enumerate(ref):
        cur = [(0, 0, r + 1)]
        for d, dec in enumerate(hypo):
            s, a, b = prev[d], cur[d], prev[d + 1]
            cur.append(min(((s[0] + (rw != dec), s[1], s[2]), (a[0], a[1] + 1, a[2]), (b[0], b[1], b[2] + 1)), key=sum))
        prev = cur
    return tuple(float(x) for x in prev[-1])


class Wer(Metric):
    """wer.py:37-117.  Lower is better; `CER` (per character) for zh / ja, else `WER`; values in percent."""

    def __init__(self, language="en"):
        super().__init__()
        self._language = language
        self._metric_key = "CER" if language in CHARACTER_LANGUAGES else "WER"

    def greater_or_eq(self, result1, result2):
        return self.get_value(result1) <= self.get_value(result2)

    def get_value(self, result):
        if isinstance(result, (float, np.float32, np.float64)):
            return result
        return result[self._metric_key]

    def _units(self, text):
        text = normalize_for_wer(self._language, text)
        return list(text.replace(" ", "")) if self._language in CHARACTER_LANGUAGES else text.split()

    def call(self, hypothesis, groundtruth):
        """Substitutions, insertions and deletions summed over the corpus, each as a share of the reference words."""
        ops, words = [0, 0, 0], 0
        for hyp, ref in zip(hypothesis, groundtruth):
            ref = self._units(ref)
            ops = [a + b for a, b in zip(ops, _wer(ref, self._units(hyp)))]
            words += len(ref)
        sub, ins, dele = (n / words for n in ops)
        k = self._metric_key
        return {k: (sub + dele + ins) * 100., k + "-substitutions": sub * 100., k + "-insertions": ins * 100.,
                k + "-deletions": dele * 100.}


# ------------------------------------------------------------------------------------------------ BLEU
def _ngram_counts(tokens, max_n):
    return Counter(tuple(tokens[i:i + n]) for n in range(1, max_n + 1) for i in range(len(tokens) - n + 1))


def _match_stats(hypotheses, references, max_n):
    """Per n-gram order the clipped matches and the hypothesis n-grams, and the corpus lengths, one reference per sentence
    (lists of tokens)."""
    matches, totals = [0] * max_n, [0] * max_n
    for hyp, ref in zip(hypotheses, references):
        h = _ngram_counts(hyp, max_n)
        for g, c in h.items():
            totals[len(g) - 1] += c
        for g, c in (h & _ngram_counts(ref, max_n)).items():
            matches[len(g) - 1] += c
    return matches, totals, sum(len(h) for h in hypotheses), sum(len(r) for r in references)


def _brevity_penalty(hyp_len, ref_len):
    return 1.0 if hyp_len >= ref_len else math.exp(1 - ref_len / hyp_len)


def tok_corpus_bleu(hypotheses, references, max_n=4):
    """Corpus BLEU in [0, 1] over whitespace tokens, without smoothing: an order without a match, or an empty
    hypothesis side, scores 0."""
    hyps, refs = [h.split() for h in hypotheses], [r.split() for r in references]
    matches, totals, hyp_len, ref_len = _match_stats(hyps, refs, max_n)
    if hyp_len == 0 or min(matches) == 0:
        return 0.0
    log_p = sum(math.log(m / t) for m, t in zip(matches, totals))
    return _brevity_penalty(hyp_len, ref_len) * math.exp(log_p / max_n)


# XML entities the reference's BLEU turns back into characters before counting, in its order ("&amp;lt;" -> "<")
XML_UNESCAPES = (("&amp;", "&"), ("&#124;", "|"), ("&lt;", "<"), ("&gt;", ">"), ("&apos;", "'"), ("&quot;", '"'),
                 ("&#91;", "["), ("&#93;", "]"))


def unescape(text):
    for entity, char in XML_UNESCAPES:
        text = text.replace(entity, char)
    return text


_RE_13A = [(re.compile(r"([\{-\~\[-\` -\&\(-\+\:-\@\/])"), r" \1 "),
           (re.compile(r"([^0-9])([\.,])"), r"\1 \2 "),
           (re.compile(r"([\.,])([^0-9])"), r" \1 \2"),
           (re.compile(r"([0-9])(-)"), r"\1 \2 ")]


def tokenize_13a(line):
    """sacrebleu's Tokenizer13a: mteval-v13a's language-independent replacements, then its punctuation regexps."""
    line = line.replace("<skipped>", "").replace("-\n", "").replace("\n", " ")
    if "&" in line:
        line = line.replace("&quot;", '"').replace("&amp;", "&").replace("&lt;", "<").replace("&gt;", ">")
    line = " %s " % line
    for pattern, repl in _RE_13A:
        line = pattern.sub(repl, line)
    return " ".join(line.split())


def sacre_corpus_bleu(hypotheses, references, lowercase=False, max_n=4):
    """sacrebleu.corpus_bleu(hypotheses, [references], lowercase, tokenize="13a").score: one reference per sentence,
    `exp` smoothing (the k-th order without a match gets precision 100 / (2^k * its n-gram count))."""
    if lowercase:
        hypotheses, references = [h.lower() for h in hypotheses], [r.lower() for r in references]
    hyps = [tokenize_13a(h.rstrip()).split() for h in hypotheses]
    refs = [tokenize_13a(r.rstrip()).split() for r in references]
    matches, totals, hyp_len, ref_len = _match_stats(hyps, refs, max_n)
    if not any(matches) or totals[-1] == 0:         # no match at all, or hypotheses too short for the highest order
        return 0.0
    log_p, halvings = 0.0, 0
    for m, t in zip(matches, totals):
        if m == 0:
            halvings += 1
            log_p += math.log(100. / (2 ** halvings * t))
        else:
            log_p += math.log(100. * m / t)
    return _brevity_penalty(hyp_len, ref_len) * math.exp(log_p / max_n)


BLEU_NAMES = ("bleu", "sacre_bleu", "tok_bleu", "detok_bleu", "uncased_sacre_bleu", "uncased_tok_bleu", "uncased_detok_bleu")


class BLEU(Metric):
    """The reference's BLEU metric without chrf, cased and uncased: `tok_bleu` is the unsmoothed corpus BLEU over the
    XML-unescaped text; `sacre_bleu` and `detok_bleu` (the same number for these languages) are sacrebleu's 13a corpus
    BLEU.  Results rank by the flag's key, else by `sacre_bleu`, so `eval_metric: bleu` keeps best by sacre_bleu."""

    def __init__(self, language="en"):
        super().__init__()
        if language in ["zh", "ja", "ko", "km", "th"]:
            raise ValueError("BLEU for language %r needs the reference's character / Thai / MeCab tokenizer, which this "
                             "path does not restate" % language)
        self._language = language

    def get_value(self, result):
        if isinstance(result, (float, np.float32, np.float64)):
            return result
        for key in (self.flag, self.flag.lower()):
            if key in result:
                return result[key]
        return result["sacre_bleu"]

    def call(self, hypothesis, groundtruth):
        out = {}
        for prefix, lc in (("", False), ("uncased_", True)):
            sacre = sacre_corpus_bleu(hypothesis, groundtruth, lowercase=lc)
            hyps, refs = ([unescape(x.lower() if lc else x) for x in side] for side in (hypothesis, groundtruth))
            out.update({prefix + "sacre_bleu": sacre, prefix + "tok_bleu": 100. * tok_corpus_bleu(hyps, refs),
                        prefix + "detok_bleu": sacre})
        return out


def check_metric_name(name):
    """The eval_metric names this path restates (case-insensitive) -> the canonical class name; others are refused."""
    low = str(name).lower()
    if low in ("wer", "cer"):
        return "wer"
    if low in BLEU_NAMES:
        return "bleu"
    if "chrf" in low:
        raise ValueError("eval_metric %r: chrf is outside this path" % name)
    raise ValueError("eval_metric %r is outside this path (wer, cer, %s)" % (name, ", ".join(BLEU_NAMES)))


def build_metric(name, language="en"):
    """build_metric(eval_metric.class, language=...): the metric object with `flag` set to the configured name, as
    SeqGenerationValidator.build does."""
    m = Wer(language) if check_metric_name(name) == "wer" else BLEU(language)
    m.flag = str(name)
    return m


# ------------------------------------------------------------------------------------------------ simultaneous latency
# Latency of the offline wait-k schedule with SimulEval's definitions (AverageLagging, AverageProportion,
# DifferentiableAverageLagging).  Units are model (BPE) tokens: |x| is the source without its EOS, |y| the hypothesis
# without its EOS, and target token i (1-based) is written after g(i) = min(k + i - 1, |x|) source tokens.  SimulEval
# reports detokenised words, so these numbers are not comparable with published word-level tables.
def waitk_delays(k, src_len, hyp_len):
    """g(i) = min(k + i - 1, |x|) for i = 1..|y|."""
    return [min(int(k) + i - 1, int(src_len)) for i in range(1, int(hyp_len) + 1)]


def simul_latency(delays, src_len):
    """{"AL", "AP", "DAL"} of one sentence from its delays g(1..|y|) and |x|; None when either side is empty.
      AL  = (1/tau) sum_{i<=tau} (g(i) - (i-1)|x|/|y|), tau the first i with g(i) = |x| (|y| when none)
      AP  = sum_i g(i) / (|x||y|)
      DAL = (1/|y|) sum_i (g'(i) - (i-1)|x|/|y|), g'(1) = g(1), g'(i) = max(g(i), g'(i-1) + |x|/|y|)"""
    x, y = int(src_len), len(delays)
    if x < 1 or y < 1:
        return None
    step = x / y
    tau = next((i + 1 for i, g in enumerate(delays) if g >= x), y)
    al = sum(delays[i] - i * step for i in range(tau)) / tau
    ap = sum(delays) / (x * y)
    dal, prev = 0.0, None
    for i, g in enumerate(delays):
        prev = g if prev is None else max(g, prev + step)
        dal += prev - i * step
    return {"AL": al, "AP": ap, "DAL": dal / y}


def waitk_latency(k, src_len, hyp_len):
    """simul_latency of the wait-k schedule (k source tokens read before the first target token, then one per token)."""
    return simul_latency(waitk_delays(k, src_len, hyp_len), src_len)


def corpus_waitk_latency(k, lengths):
    """Means of AL / AP / DAL over (|x|, |y|) pairs, skipping sentences with an empty side; None when none is left."""
    rows = [r for r in (waitk_latency(k, x, y) for x, y in lengths) if r is not None]
    if not rows:
        return None
    return {m: sum(r[m] for r in rows) / len(rows) for m in ("AL", "AP", "DAL")}
