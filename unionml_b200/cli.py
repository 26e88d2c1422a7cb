"""``serve`` launcher: ``python -m unionml_b200.cli serve app:app --model-path model.joblib [uvicorn options]``.

The reference's ``unionml serve`` (``unionml:unionml/cli.py:285-320``) is uvicorn's own CLI with one extra option,
``--model-path``, exported to the app as ``UNIONML_MODEL_PATH`` before uvicorn starts (the FastAPI startup hook loads the
model from it, ``unionml/fastapi.py:22-34``).  Same here; the other reference commands (``init / deploy / train /
predict / list-* / fetch-*``) talk to a Flyte cluster and are out of scope.  The CUDA engine is bound lazily by the
first ``/predict`` in each worker process, never here (uvicorn ``--workers`` forks).
"""
import argparse
import os
import sys


def main(argv=None) -> int:
    parser = argparse.ArgumentParser(prog="unionml_b200")
    sub = parser.add_subparsers(dest="command", required=True)
    serve = sub.add_parser("serve", help="start a prediction server (uvicorn) for a unionml_b200 app")
    serve.add_argument("app", help="ASGI app as module:attribute, e.g. app:app")
    serve.add_argument("--model-path", default=None, help="saved model object (exported as UNIONML_MODEL_PATH)")
    serve.add_argument("--host", default="127.0.0.1")
    serve.add_argument("--port", type=int, default=8000)
    serve.add_argument("--workers", type=int, default=None)
    serve.add_argument("--reload", action="store_true")
    serve.add_argument("--log-level", default="info")
    args = parser.parse_args(argv)

    if args.command == "serve":
        if args.model_path is not None:
            if not os.path.exists(args.model_path):
                parser.error(f"model path {args.model_path} not found")
            os.environ["UNIONML_MODEL_PATH"] = str(args.model_path)
        import uvicorn

        sys.path.insert(0, os.getcwd())
        uvicorn.run(args.app, host=args.host, port=args.port, workers=args.workers, reload=args.reload,
                    log_level=args.log_level)
    return 0


if __name__ == "__main__":
    sys.exit(main())
