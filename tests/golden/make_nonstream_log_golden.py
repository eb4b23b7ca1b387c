"""Generates tests/golden/nonstream_log_cases.json: the log files and usage rows the UNMODIFIED reference middleware
(llm_gateway_core/middleware/chat_logging.py:22-67, :87-150, :165-231, registered with app.middleware("http") as main.py does)
leaves for non-streaming responses of /v1/chat/completions, in the order they happen.  Dev-container only (reads the reference);
the committed JSON is what the tests use.

    python tests/golden/make_nonstream_log_golden.py

The clock of write_log is tests/nonstream_log_cases.Clock and the row insert is a recorder, as in make_write_log_golden.py.  The
tap thread waits 2 s on its queue before its final write_log (:100): it is joined before the log directory is read.
"""
import base64
import json
import os
import sys
import tempfile
import threading
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
import ref_driver
import nonstream_log_cases as nc


def main():
    _, cl = ref_driver.load_reference()
    real_insert, real_dt = cl.tokens_usage_db.insert_usage, cl.datetime
    cwd = os.getcwd()
    out = []
    for case in nc.cases():
        with tempfile.TemporaryDirectory() as d:
            os.chdir(d)
            rec = nc.Recorder(Path(d, "logs"))
            cl.tokens_usage_db.insert_usage = rec
            cl.datetime = nc.Clock()                                        # write_log calls datetime.now() (:25)
            try:
                status, body = nc.post(case, cl.log_chat_completions)
                for t in threading.enumerate():
                    if isinstance(t, cl.ChunkProcessorThread):
                        t.join()
                events = rec.finish()
            finally:
                cl.tokens_usage_db.insert_usage, cl.datetime = real_insert, real_dt
                os.chdir(cwd)
        g = dict(name=case["name"], kind=case["kind"], request=base64.b64encode(case["request"]).decode())
        if case["kind"] == "doc":
            g["doc"] = base64.b64encode(case["doc"]).decode()
        else:
            g.update(status=case["status"], detail=case["detail"])
        g.update(response_status=status, response=base64.b64encode(body).decode(), events=nc.encode_events(events))
        out.append(g)
        print(case["name"], status, [e[0] for e in events])
    doc = dict(generator="tests/golden/make_nonstream_log_golden.py",
               reference="llm_gateway_core/middleware/chat_logging.py (unmodified), app.middleware('http')", cases=out)
    (HERE / "nonstream_log_cases.json").write_text(json.dumps(doc, indent=1, ensure_ascii=True))
    print(len(out), "cases")


if __name__ == "__main__":
    main()
