"""FastAPI application: V1, V2 and OpenAI routes + error handlers + /metrics (mirrors
python/kserve/kserve/protocol/rest/server.py:56-189, v1_endpoints.py:33-174, v2_endpoints.py:35-305)."""
from __future__ import annotations

from typing import Any, AsyncIterator, Dict, Optional, Tuple

from fastapi import FastAPI, Request, Response
from fastapi.responses import JSONResponse, StreamingResponse
from prometheus_client import CONTENT_TYPE_LATEST, generate_latest

from ... import errors as E
from ..dataplane import DataPlane
from .openai.dataplane import OpenAIDataPlane
from .openai.endpoints import register_openai_endpoints
from .openai.openai_model import OpenAIModel


def create_application(dataplane: OpenAIDataPlane, batcher: Optional[Tuple[int, int]] = None) -> FastAPI:
    """batcher = (max_batchsize, max_latency_ms) installs the request batcher in front of V1 `:predict`, where the Go
    agent puts it (cmd/agent/main.go:256-273 startBatcher, :431-433 `batcher.New(...)` wrapping the proxy to the model
    server; pkg/batcher/handler.go:222-266 ServeHTTP).  Concurrent `:predict` requests are merged into ONE downstream
    predict whose instances are the concatenation of theirs; every caller gets `{"message", "batchId", "predictions"}`
    with its own slice."""
    app = FastAPI(title="KServe ModelServer (H100 runtime)", version=dataplane._server_version)
    dp: DataPlane = dataplane
    batch_handler = None
    if batcher is not None:
        from ....batcher import BatchHandler

        async def downstream(path: str, body: Dict[str, Any]) -> Tuple[int, Any]:
            """the predictor behind the batcher: what the agent's reverse proxy reaches over HTTP, called in-process"""
            model_name = path.rsplit("/", 1)[-1].rsplit(":", 1)[0]
            try:
                response, _ = await dp.infer(model_name=model_name, request=body, headers={})
            except E.InvalidInput as e:
                return 400, {"error": str(e)}
            except E.ModelNotFound as e:
                return 404, {"error": str(e)}
            except E.ModelNotReady as e:
                return 503, {"error": str(e)}
            except Exception as e:   # InferenceError and anything else: a 500 from the predictor
                return 500, {"error": f"{type(e).__name__} : {e}"}
            return 200, response
        batch_handler = BatchHandler(batcher[0], batcher[1], downstream)
        app.state.batch_handler = batch_handler

    # ---- health / metadata
    @app.get("/")
    async def live():
        return await dp.live()

    @app.get("/metrics")
    async def metrics():
        return Response(generate_latest(), media_type=CONTENT_TYPE_LATEST)

    @app.get("/v1/models")
    async def v1_models():
        return {"models": list(dp.model_registry.get_models().keys())}

    @app.get("/v1/models/{model_name}")
    async def v1_model_ready(model_name: str):
        if not await dp.model_ready(model_name):
            raise E.ModelNotReady(model_name)
        return {"name": model_name, "ready": True}

    @app.get("/v2")
    async def v2_metadata():
        return dp.metadata()

    @app.get("/v2/health/live")
    async def v2_live():
        return {"live": True}

    @app.get("/v2/health/ready")
    async def v2_ready():
        return {"ready": await dp.ready()}

    @app.get("/v2/models/{model_name}")
    async def v2_model_metadata(model_name: str):
        return await dp.model_metadata(model_name)

    @app.get("/v2/models/{model_name}/ready")
    async def v2_model_ready(model_name: str):
        if not await dp.model_ready(model_name):
            raise E.ModelNotReady(model_name)
        return {"name": model_name, "ready": True}

    # ---- V1 predict (v1_endpoints.py:61-100)
    @app.post("/v1/models/{model_name}:predict")
    async def v1_predict(model_name: str, request: Request):
        if not await dp.model_ready(model_name, True):
            raise E.ModelNotReady(model_name)
        body = await request.body()
        if batch_handler is not None:        # handler.go:222-266
            status, out = await batch_handler.serve(request.url.path, body)
            if status != 200 or isinstance(out, str):
                return Response(content=(out if isinstance(out, str) else str(out)) + "\n", status_code=status,
                                media_type="text/plain; charset=utf-8")     # http.Error(w, msg, code)
            return JSONResponse(content=out)
        headers = dict(request.headers.items())
        infer_request, attrs = dp.decode(body=body, headers=headers)
        response, response_headers = await dp.infer(model_name=model_name, request=infer_request, headers=headers)
        response, res_headers = dp.encode(model_name=model_name, response=response, headers=headers, req_attributes=attrs)
        response_headers.update(res_headers)
        response_headers.pop("content-length", None)
        if isinstance(response, (bytes, str)):
            return Response(content=response, headers=response_headers)
        if isinstance(response, AsyncIterator):
            return StreamingResponse(content=response)
        return JSONResponse(content=response, headers=response_headers)

    # ---- V1 explain (v1_endpoints.py:102-140): the predict route with the EXPLAIN verb
    @app.post("/v1/models/{model_name}:explain")
    async def v1_explain(model_name: str, request: Request):
        if not await dp.model_ready(model_name, True):
            raise E.ModelNotReady(model_name)
        body = await request.body()
        headers = dict(request.headers.items())
        infer_request, attrs = dp.decode(body=body, headers=headers)
        response, response_headers = await dp.explain(model_name=model_name, request=infer_request, headers=headers)
        response, res_headers = dp.encode(model_name=model_name, response=response, headers=headers, req_attributes=attrs)
        response_headers.update(res_headers)
        response_headers.pop("content-length", None)
        if isinstance(response, (bytes, str)):
            return Response(content=response, headers=response_headers)
        return JSONResponse(content=response, headers=response_headers)

    @app.get("/v2/models")
    async def v2_models():
        return {"models": list(dp.model_registry.get_models().keys())}

    # ---- V2 infer (v2_endpoints.py:132-194)
    @app.post("/v2/models/{model_name}/infer")
    async def v2_infer(model_name: str, request: Request):
        if not await dp.model_ready(model_name, True):
            raise E.ModelNotReady(model_name)
        headers = dict(request.headers)
        body = await request.body()
        infer_request, _ = dp.decode(body, headers, protocol_version="v2", model_name=model_name)
        response, response_headers = await dp.infer(model_name=model_name, request=infer_request, headers=headers)
        response, res_headers = dp.encode(model_name=model_name, response=response, headers=headers, req_attributes={})
        response_headers.update(res_headers)
        response_headers.pop("content-length", None)
        if isinstance(response, bytes):
            return Response(content=response, headers=response_headers, media_type="application/octet-stream")
        response_headers.pop("content-type", None)
        # JSON-only responses go through the reference's pydantic `InferenceResponse` (v2_datamodels.py): fixed key order
        # model_name, model_version, id, parameters, outputs[name, shape, datatype, parameters, data], absent values as
        # null (byte strings pinned by test_server.py:591-632, :744-778)
        if isinstance(response, dict) and "outputs" in response:
            response = {"model_name": response.get("model_name"), "model_version": response.get("model_version"),
                        "id": response.get("id"), "parameters": response.get("parameters"),
                        "outputs": [{"name": o.get("name"), "shape": o.get("shape"), "datatype": o.get("datatype"),
                                     "parameters": o.get("parameters"), "data": o.get("data")} for o in response["outputs"]]}
        return JSONResponse(content=response, headers=response_headers)

    # ---- error handlers (rest/server.py:134-145)
    app.add_exception_handler(E.InvalidInput, E.invalid_input_handler)
    app.add_exception_handler(E.InferenceError, E.inference_error_handler)
    app.add_exception_handler(E.ModelNotFound, E.model_not_found_handler)
    app.add_exception_handler(E.ModelNotReady, E.model_not_ready_handler)
    app.add_exception_handler(NotImplementedError, E.not_implemented_error_handler)
    app.add_exception_handler(E.UnsupportedProtocol, E.unsupported_protocol_error_handler)
    app.add_exception_handler(E.ServerNotReady, E.server_not_ready_handler)
    app.add_exception_handler(Exception, E.generic_exception_handler)

    # OpenAI routes only if an OpenAIModel is registered (openai/config.py:21-46)
    if any(isinstance(m, OpenAIModel) for m in dp.model_registry.get_models().values()):
        register_openai_endpoints(app, dataplane)
    return app
