"""networks.evaluator (reference networks/evaluator.py): the Hungarian-matched instance loss of the training step
(ins_criterion / hungarian) and the small loss lambdas run on the native kernels; the evaluation-time metrics (ins_eval,
calculate_ap) are re-exported from the reference checkout when DMNERF_REFERENCE_ROOT points at one, and are the native
device versions (dmnerf_b200.tester) otherwise."""
import importlib.util as _ilu
import os as _os

_ref = _os.environ.get("DMNERF_REFERENCE_ROOT")
if _ref and _os.path.exists(_os.path.join(_ref, "networks", "evaluator.py")):
    _spec = _ilu.spec_from_file_location("_dmnerf_reference_evaluator", _os.path.join(_ref, "networks", "evaluator.py"))
    _mod = _ilu.module_from_spec(_spec)
    _spec.loader.exec_module(_mod)
    globals().update({k: v for k, v in vars(_mod).items() if not k.startswith("__")})

from dmnerf_b200.evaluator import ins_criterion, img2mse, mse2psnr, to8b   # noqa: F401,E402

# ins_eval (test-time metrics on CPU tensors) keeps calling the reference's own CPU `hungarian` through its module globals;
# the training-time entry point ins_criterion is the native one for every importer of this module.
if "_mod" in globals():
    _mod.ins_criterion = ins_criterion
else:
    from dmnerf_b200.evaluator import hungarian   # noqa: F401,E402
    from dmnerf_b200.tester import ins_eval, calculate_ap   # noqa: F401,E402
