"""Cooperative stop flag (capability parity with scaelum/runner/hooks_collection/stop_hook.py:
12-38, with the attribute bugs of SURVEY §2.7 fixed).

``before_run`` writes "0" to ``<root>/stop_flag.txt`` (rank 0 only), ``after_iter`` makes every
rank agree on the flag (rank 0 reads the file, the value is broadcast) and, on "1", pushes
iter/epoch past their maxima; ``StopHook.stop(root)`` is the external trigger.
"""
import os
import os.path as osp

from ...registry import HOOKS
from ..hooks import Hook


def _dist():
    import torch.distributed as dist

    return dist if dist.is_available() and dist.is_initialized() else None


@HOOKS.register_module
class StopHook(Hook):
    def __init__(self, root="/tmp", check_interval: int = 1):
        super().__init__()
        self.root = root
        self.file_path = osp.join(root, "stop_flag.txt")
        self.check_interval = check_interval

    def _is_rank0(self):
        d = _dist()
        return d is None or d.get_rank() == 0

    def before_run(self, runner):
        if self._is_rank0():
            os.makedirs(self.root, exist_ok=True)
            with open(self.file_path, "w") as f:
                f.write("0")

    def after_iter(self, runner):
        if not self.every_n_iters(runner, self.check_interval):
            return
        flag = "0"
        if self._is_rank0() and osp.exists(self.file_path):
            with open(self.file_path, "r") as f:
                flag = f.readline().strip()
        d = _dist()
        if d is not None and d.get_world_size() > 1:
            obj = [flag]
            d.broadcast_object_list(obj, src=0)
            flag = obj[0]
        if flag == "1":
            runner.request_stop()

    def after_val_iter(self, runner):
        # the flag is checked between training iterations only
        return None

    def after_run(self, runner):
        if self._is_rank0() and osp.exists(self.file_path):
            os.remove(self.file_path)

    @staticmethod
    def stop(root):
        with open(osp.join(root, "stop_flag.txt"), "w") as f:
            f.write("1")
