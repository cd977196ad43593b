"""Import the UNMODIFIED reference implementation: the checkout named by OVC_REFERENCE, else the file-by-file copy
under oracle/_ref/ (oracle/make_ref.py; git-ignored).  Without either, the ``reference``-marked tests skip.

TEST / MEASUREMENT INFRASTRUCTURE.  Used by tools/make_golden.py to generate the fixtures under tests/golden/,
by the ``reference``-marked tests that compare against the live reference, and by oracle/ref_python_bench.py
(bench.py's `cpu_baseline.reference_python`: the reference's own Python step timed on the box's host cores).
Nothing on the ``-m gpu`` / smoke path imports this.

Follows SURVEY.md appendix E: stub the four optional modules the reference imports at module
scope (gymnasium, pygame, IPython, ipywidgets), never let the planners write pickles into the
read-only reference tree, never write bytecode there.
"""
import os
import sys
import types

_HERE = os.path.dirname(os.path.abspath(__file__))


def _find_root():
    """OVC_REFERENCE (a checkout of the reference repository), else the copy oracle/make_ref.py made."""
    return os.environ.get("OVC_REFERENCE") or os.path.join(_HERE, "_ref")


REFERENCE_ROOT = _find_root()


def available():
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "src", "overcooked_ai_py"))


class _Dummy(types.ModuleType):
    """A module whose every attribute is another dummy (callable, subclassable)."""

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        sub = _DummyObj()
        setattr(self, name, sub)
        return sub


class _DummyObj(object):
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _DummyObj()

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return _DummyObj()

    def __iter__(self):
        return iter(())

    def __getitem__(self, k):
        return _DummyObj()

    def __mro_entries__(self, bases):  # lets `class X(dummy.Base)` work
        return (object,)


_BOOTED = None


def boot():
    """Returns a namespace with the reference's mdp / env / planner / agent modules."""
    global _BOOTED
    if _BOOTED is not None:
        return _BOOTED
    if not available():
        raise RuntimeError("reference tree not found at %s" % REFERENCE_ROOT)
    sys.dont_write_bytecode = True
    for name in (
        "gymnasium", "gymnasium.spaces", "gymnasium.envs", "gymnasium.envs.registration",
        "pygame", "pygame.locals", "IPython", "IPython.display", "ipywidgets",
    ):
        if name not in sys.modules:
            sys.modules[name] = _Dummy(name)
    sys.modules["gymnasium"].Env = object
    sys.modules["gymnasium.envs.registration"].register = lambda *a, **k: None
    src = os.path.join(REFERENCE_ROOT, "src")
    if src not in sys.path:
        sys.path.insert(0, src)
    import overcooked_ai_py.agents.agent as agent
    import overcooked_ai_py.mdp.actions as actions
    import overcooked_ai_py.mdp.overcooked_env as env
    import overcooked_ai_py.mdp.overcooked_mdp as mdp
    import overcooked_ai_py.planning.planners as planners

    # the planners pickle themselves into the package data dir on compute: forbid it
    planners.MotionPlanner.save_to_file = lambda self, filename: None
    planners.MediumLevelActionManager.save_to_file = lambda self, filename: None
    for cls_name in ("JointMotionPlanner", "MediumLevelPlanner"):
        cls = getattr(planners, cls_name, None)
        if cls is not None and hasattr(cls, "save_to_file"):
            cls.save_to_file = lambda self, filename: None

    ns = types.SimpleNamespace(mdp=mdp, env=env, actions=actions, planners=planners, agent=agent)
    _BOOTED = ns
    return ns


def make_mdp(ns, layout_name, **params):
    """A reference OvercookedGridworld.  The reference keeps recipe values in CLASS state
    (Recipe.configure, overcooked_mdp.py:220-336, quirk Q1), so re-configure before every use."""
    m = ns.mdp.OvercookedGridworld.from_layout_name(layout_name, **params)
    return m


def use_mdp(ns, m):
    ns.mdp.Recipe.configure(m.recipe_config)
    return m


def make_env(ns, m, horizon=400, start_state_fn=None):
    use_mdp(ns, m)
    e = ns.env.OvercookedEnv.from_mdp(m, horizon=horizon, info_level=0, start_state_fn=start_state_fn)
    e._mp = object()  # never build / pickle a MotionPlanner for step-only use (overcooked_env.py:258)
    return e


class LitePlannerHolder(object):
    """featurize_state only reads ``mlam.motion_planner`` (overcooked_mdp.py:2822,2901)."""

    def __init__(self, ns, m):
        use_mdp(ns, m)
        self.motion_planner = ns.planners.MotionPlanner(m)
