"""CPU checks of which driver runs an adaptive solve (_engine.choose_driver): the whole decision table against the
selection the engine made before the choice was one function, and the engine's facts as _plan reads them."""
import itertools

from torchdiffeq_b200._engine import AdaptiveEngine, choose_driver

OPTION = (True, False, "auto")
FACTS = dict(lockstep=(True, False), fused_solve=(True, False), device_loop=OPTION, agree_fn=(True, False),
             norm_fn=(True, False), exchange=(True, False), keep_interp=(True, False), has_loop=(True, False),
             has_graph=(True, False), graph=OPTION, graph_failed=(True, False), capture_in_solve=(True, False))


def _reference(lockstep, fused_solve, device_loop, agree_fn, norm_fn, exchange, keep_interp, has_loop, has_graph,
               graph, graph_failed, capture_in_solve):
    """The earlier selection, condition by condition: solve() took lock step on _lockstep_mode(); _loop_run_ahead()
    then tried _linear_solve_ready(), launched the loop on _use_loop() (its handle armed by _begin on the same test),
    and without a graph ran attempt 1 eagerly, capturing it when use_graph held; anything else replayed or ran eagerly."""
    if lockstep:
        return "lockstep"
    linear_solve_ready = (fused_solve and device_loop in (True, "auto") and not lockstep and not agree_fn
                          and not norm_fn and not exchange and not keep_interp)
    if linear_solve_ready:
        return "persistent"
    use_loop = has_loop and not lockstep and not agree_fn and not norm_fn
    if use_loop:
        return "loop"
    use_graph = graph in (True, "auto") and not graph_failed and capture_in_solve
    if not has_graph:
        return "capture" if use_graph else "eager"
    return "replay"


def test_decision_table_matches_the_earlier_selection():
    names = list(FACTS)
    seen = set()
    for values in itertools.product(*FACTS.values()):
        facts = dict(zip(names, values))
        got = choose_driver(**facts)
        assert got == _reference(**facts), facts
        seen.add(got)
    assert seen == {"lockstep", "persistent", "loop", "replay", "capture", "eager"}


# a fused linear solve that may run as one persistent launch, before anything was captured
FUSED = dict(lockstep=False, fused_solve=True, device_loop="auto", agree_fn=False, norm_fn=False, exchange=False,
             keep_interp=False, has_loop=False, has_graph=False, graph="auto", graph_failed=False, capture_in_solve=True)


def test_refused_persistent_launch_falls_back_to_the_per_attempt_choice():
    assert choose_driver(**FUSED) == "persistent"
    # the device refused the cooperative launch: the same solve captures, and later solves use what it captured
    refused = dict(FUSED, fused_solve=False)
    assert choose_driver(**refused) == "capture"
    assert choose_driver(**dict(refused, has_graph=True, has_loop=True)) == "loop"
    assert choose_driver(**dict(refused, graph=False)) == "eager"


def test_capture_then_loop():
    first = dict(FUSED, fused_solve=False)
    assert choose_driver(**first) == "capture"
    assert choose_driver(**dict(first, has_graph=True, has_loop=True)) == "loop"        # the capture made a loop
    assert choose_driver(**dict(first, has_graph=True)) == "replay"                     # it did not
    assert choose_driver(**dict(first, has_graph=True, has_loop=True, agree_fn=True)) == "replay"
    assert choose_driver(**dict(first, graph_failed=True)) == "eager"
    assert choose_driver(**dict(first, capture_in_solve=False)) == "eager"              # the adjoint's backward solve


def _parent_engine_choice(e):
    """The earlier engine methods on the same attributes: _lockstep_mode(), _linear_solve_ready(), _use_loop() and
    _loop_run_ahead()'s use_graph."""
    lockstep = bool(e.callbacks) or e.run_ahead == 0
    L = e.linear
    if lockstep:
        return "lockstep"
    if (L is not None and L["whole"] and L["fold"] and not e._solve_refused and e.device_loop in (True, "auto")
            and e.agree_fn is None and e.norm_fn is None and e.exchange is None and not e.keep_interp):
        return "persistent"
    if e._loop is not None and e.agree_fn is None and e.norm_fn is None:
        return "loop"
    if e._graph is None:
        use_graph = e.graph_opt in (True, "auto") and not e._graph_failed and e.capture_in_solve
        return "capture" if use_graph else "eager"
    return "replay"


def test_plan_reads_the_engine():
    """_plan() maps the engine's attributes to the facts as the earlier methods read them (callbacks always come with
    run_ahead = 0), and prime() captures where a solve would, whatever capture_in_solve says."""
    linears = [None, dict(whole=False, fold=False), dict(whole=True, fold=False), dict(whole=True, fold=True)]
    host = [None, "agree_fn", "norm_fn", "exchange"]
    held = [(None, None), (object(), None), (object(), 1)]
    for linear, run_ahead, refused, capture_in_solve, hosted, (graph, loop), keep_interp in itertools.product(
            linears, (0, 2), (False, True), (False, True), host, held, (False, True)):
        eng = AdaptiveEngine.__new__(AdaptiveEngine)
        eng.callbacks, eng.run_ahead, eng.linear, eng._solve_refused = {}, run_ahead, linear, refused
        eng.agree_fn = eng.norm_fn = eng.exchange = None
        if hosted is not None:
            setattr(eng, hosted, object())
        eng.device_loop, eng.keep_interp, eng._graph, eng._loop = "auto", keep_interp, graph, loop
        eng.graph_opt, eng._graph_failed, eng.capture_in_solve = "auto", False, capture_in_solve
        want = _parent_engine_choice(eng)
        assert eng._plan() == want, (linear, run_ahead, refused, capture_in_solve, hosted, graph, loop, keep_interp)
        eng.capture_in_solve = True
        assert eng._plan(priming=True) == _parent_engine_choice(eng)
