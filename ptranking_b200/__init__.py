"""ptranking_b200 -- H100-native (sm_90a) scoring-and-loss hot path behind PTRanking's plugin API.

    import ptranking_b200
    ptranking_b200.install()           # swap the loss classes into ptranking.ltr_adhoc.eval.ltr
    LTREvaluator(cuda=0).run(model_id='LambdaRank', ...)   # the unmodified reference driver

    ptranking_b200.install_diversification()   # DALETOR and DivProbRanker into ptranking.ltr_diversification.eval.ltr_diversification
    DivLTREvaluator(cuda=0).run(model_id='DALETOR', sf_id='pointsf', ...)

    ptranking_b200.install_data()      # opt-in: LTRDataset reads the LETOR files on the device (read_letor)

Importing the package never touches the GPU; the first kernel call loads
lib/libptranking_b200.so and raises if it (or an sm_90 device) is missing.
"""
from .ltr_adhoc.pairwise.ranknet import RankNet
from .ltr_adhoc.listwise.lambdarank import LambdaRank
from .ltr_adhoc.listwise.lambdaloss import LambdaLoss
from .ltr_adhoc.listwise.listnet import ListNet
from .ltr_adhoc.listwise.listmle import ListMLE
from .ltr_adhoc.listwise.approxNDCG import ApproxNDCG
from .ltr_adhoc.pointwise.rank_mse import RankMSE
from .ltr_adhoc.listwise.rank_cosine import RankCosine
from .ltr_adhoc.listwise.st_listnet import STListNet
from .ltr_adhoc.listwise.softrank import SoftRank
from .ltr_adhoc.listwise.wassrank import WassRank
from .ltr_adhoc.listwise.mdprank import MDPRank
from .ltr_diversification.score_and_sort.daletor import DALETOR
from .ltr_diversification.score_and_sort.div_prob_ranker import DivProbRanker
from .base.ranker import LABEL_TYPE
from .letor import LetorSplit, LTRDataset, read_letor

MODELS = {c.__name__: c for c in (RankNet, LambdaRank, LambdaLoss, ListNet, ListMLE, ApproxNDCG,
                                  RankMSE, RankCosine, STListNet, SoftRank, WassRank, MDPRank)}
DIV_MODELS = {c.__name__: c for c in (DALETOR, DivProbRanker)}
__version__ = "0.1.0"


def install(module=None):
    """Register the CUDA classes where the reference resolves model ids by name:
    ``globals()[model_id]`` in ptranking/ltr_adhoc/eval/ltr.py:166-171."""
    if module is None:
        import ptranking.ltr_adhoc.eval.ltr as module  # the reference package must be importable
    previous = {}
    for name, cls in MODELS.items():
        previous[name] = getattr(module, name, None)
        setattr(module, name, cls)
    # The driver also looks up globals()[model_id + "Parameter"] (ltr.py:463), and the reference's ltr.py imports no
    # MDPRankParameter: supply the reference's own class, when its module is importable.
    if getattr(module, 'MDPRankParameter', None) is None:
        try:
            from ptranking.ltr_adhoc.listwise.mdprank import MDPRankParameter
        except ImportError:
            pass
        else:
            previous['MDPRankParameter'] = getattr(module, 'MDPRankParameter', None)
            setattr(module, 'MDPRankParameter', MDPRankParameter)
    return previous


def install_diversification(module=None):
    """Register the diversification classes where the reference's diversification driver resolves model ids by name:
    ``globals()[model_id]`` in ptranking/ltr_diversification/eval/ltr_diversification.py:385-389.  Returns
    {name: the value it replaced} for the names the module already had (the reference's driver has all of them)."""
    if module is None:
        import ptranking.ltr_diversification.eval.ltr_diversification as module  # the reference must be importable
    previous = {}
    for name, cls in DIV_MODELS.items():
        if hasattr(module, name):
            previous[name] = getattr(module, name)
        setattr(module, name, cls)
    return previous


def install_data(module=None):
    """Opt-in: make the reference driver load its splits with :class:`ptranking_b200.letor.LTRDataset`, which parses
    the LETOR files on the device (``LTRDataset(...)`` in ptranking/ltr_adhoc/eval/ltr.py:138-148).  ``install()`` does
    not call this.  Returns {name: the value it replaced}."""
    if module is None:
        import ptranking.ltr_adhoc.eval.ltr as module  # the reference package must be importable
    previous = {"LTRDataset": getattr(module, "LTRDataset", None)}
    module.LTRDataset = LTRDataset
    return previous
