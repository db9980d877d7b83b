"""The card a developer benchmark ran on, read in the same run as its numbers: an absolute time or rate means little
without the card's name and its power limit (a card set below 700 W lowers its clocks under sustained load)."""
import subprocess
import torch


def card():
    """torch's name for device 0, and nvidia-smi's read-only query of its name, power limit and maximum SM clock, or
    'unavailable' where nvidia-smi is missing or fails (the numbers stay valid without it; nothing is raised)."""
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30,
                           check=True).stdout.decode().strip()
    except (OSError, subprocess.SubprocessError):
        q = ''
    return dict(name=torch.cuda.get_device_name(0), nvidia_smi=q or 'unavailable')
