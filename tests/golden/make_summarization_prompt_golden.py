"""Generate tests/golden/summarization_prompts.json: prompts the REFERENCE's summarization mode receives, recorded from its
R2R agent (tasks/agents/r2r.py R2RAgent.get_summarization_prompt) for a few history / candidate counts.

    NAVILLM_REFERENCE=<reference checkout> python tests/golden/make_summarization_prompt_golden.py

tools/diverse_beam_bench.py builds its summarization-shaped batch from these recorded prompts (nothing reads the reference at
run time).
"""
import json
import os
import sys
from pathlib import Path

REF = os.environ["NAVILLM_REFERENCE"]
SIZES = [(7, 6), (5, 4), (10, 8)]                  # (history steps, candidates): a typical R2R path, a short and a long one


def main():
    sys.path.insert(0, REF)
    from tasks.agents.r2r import R2RAgent
    out = {"source": "tasks/agents/r2r.py R2RAgent.get_summarization_prompt(instruction, hist_num, cand_num)",
           "prompts": [{"hist_num": h, "cand_num": c, "prompt": R2RAgent.get_summarization_prompt(None, "", h, c)}
                       for h, c in SIZES]}
    path = Path(__file__).resolve().parent / "summarization_prompts.json"
    path.write_text(json.dumps(out, indent=1) + "\n")
    print(path)


if __name__ == "__main__":
    main()
