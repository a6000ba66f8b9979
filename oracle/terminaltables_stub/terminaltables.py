class AsciiTable:  # utils/prune_utils.py imports it only to print tables
    def __init__(self, data): self.table = "\n".join(" ".join(str(c) for c in row) for row in data)
