"""`models` package name of the reference checkout, resolved to the H100 engine (see compat/README.md)."""
