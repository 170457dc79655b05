"""`python -m localexpstereo_b200 -mode MiddV2|MiddV3 -targetDir D -outputDir O [...]`: the reference's command (see cli.py)."""
import sys

from .cli import main

sys.exit(main())
