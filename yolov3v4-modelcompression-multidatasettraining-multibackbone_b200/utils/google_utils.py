"""Download helpers of the reference (utils/google_utils.py) are out of scope (no network on the target box).
Only the names models.py star-imports are kept so that `from models import *` behaves the same."""
import os
import time


def gdrive_download(id='', name=''):
    raise RuntimeError("gdrive_download(%r): network downloads are not part of the H100 hot path" % name)


def upload_blob(*a, **k):
    raise RuntimeError("GCS upload is not part of the H100 hot path")


def download_blob(*a, **k):
    raise RuntimeError("GCS download is not part of the H100 hot path")
