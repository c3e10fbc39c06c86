"""Process-global communication timer (mirrors PipeGCN/helper/timer/timer.py:3)."""
from .comm_timer import CommTimer

comm_timer = CommTimer()
