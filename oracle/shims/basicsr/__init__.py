"""Import shim (test infrastructure only): stands in for the `basicsr` package so the
read-only reference checkout (oracle/reference_loader.py) can be imported as a CPU oracle. Not product code."""
