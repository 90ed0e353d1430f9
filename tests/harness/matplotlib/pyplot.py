"""Empty stand-in (see __init__.py)."""
