# Build + CPU test image.  Run the GPU tiers with `docker run --gpus all` on a H100 host.
FROM nvidia/cuda:12.9.0-devel-ubuntu24.04
ENV DEBIAN_FRONTEND=noninteractive
RUN apt-get update && apt-get install -y --no-install-recommends python3 python3-pip python3-venv git build-essential \
    && rm -rf /var/lib/apt/lists/*
RUN python3 -m venv /opt/venv
ENV PATH=/opt/venv/bin:$PATH
RUN pip install --no-cache-dir torch numpy scipy pybind11 pytest
WORKDIR /opt/sparkflow_b200
COPY . .
RUN python tools/build_ext.py
CMD ["python", "-m", "pytest", "tests", "-q", "-m", "not gpu"]
